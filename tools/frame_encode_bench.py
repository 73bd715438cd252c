"""Device LZ4 Frame writer (b200lz4f_compress_dev) against its floor and against what a caller with device-resident data does
without it, on one GPU.

The data: RDG P=0.5 (the bench corpus) from a seeded 256 MiB host sample, tiled across --gib GiB of device memory with the
first 8 bytes of every 64 KiB perturbed so that blocks differ.  It is split four ways: 1 frame, 64 frames, 4096 frames, and
4096 frames of mixed sizes.  Each split runs at bsCode 4 and 7 with flags 0 (nothing), 2 (block checksums) and 1 (content
checksum), and three things are timed, alternately in the same process, median of --runs after a warm-up:
  dev    b200lz4f_compress_dev over the split                                             (CUDA events)
  floor  b200lz4_compress_fast_batch_dev over the same blocks into bound-sized slots      (CUDA events)
  host   the source copied to pinned host memory, then b200lz4f_compress_host per frame   (wall clock), over the first
         --host-gib GiB of the split's frames, since it needs that much pinned and pageable host memory three times over
The device writer's output on the host leg's frames is compared with the host writer's by digest.
    python tools/frame_encode_bench.py [--gib 16] [--runs 5] [--host-gib 1] [--host-runs 2]
"""
import argparse
import hashlib
import json
import subprocess
import sys
import time

import _variant  # noqa: F401  (B200LZ4_TEST_SO: another build of the library)
import numpy as np


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def splits(total, rng):
    one = [total]
    s64 = [total // 64] * 64
    s64[-1] += total - sum(s64)
    s4k = [total // 4096] * 4096
    s4k[-1] += total - sum(s4k)
    w = rng.lognormal(0.0, 1.5, 4096)
    mixed = np.maximum((w / w.sum() * total).astype(np.int64), 1)
    mixed[-1] += total - int(mixed.sum())
    return {"1 frame": one, "64 frames": s64, "4096 frames": s4k, "4096 mixed": [int(x) for x in mixed]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=16)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--host-gib", type=float, default=1)
    ap.add_argument("--host-runs", type=int, default=2)
    ap.add_argument("--seed", type=int, default=2)
    ap.add_argument("--json", default="", help="also append every result to this file, one JSON line each")
    args = ap.parse_args()

    import torch
    import lz4java_b200 as L
    from oracle import oracle as O
    lib = L._native.lib()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)

    BLK = 65536
    total = int(args.gib * (1 << 30)) // BLK * BLK
    base_n = min(total, 256 << 20)
    base = torch.from_numpy(O.best_available().datagen(base_n, 0.5, 0.0, args.seed)).to(dev)
    src = torch.empty(total, dtype=torch.uint8, device=dev)
    for lo in range(0, total, base_n):
        src[lo:lo + base_n] = base[:min(base_n, total - lo)]
    nblk = total // BLK
    idx = torch.arange(nblk, device=dev, dtype=torch.int64)
    v = src.view(nblk, BLK)
    for k in range(8):
        v[:, k] ^= ((idx >> (8 * k)) & 0xFF).to(torch.uint8)
    del base, idx, v
    dst_cap = total + total // 255 + 32 * (nblk + 4096) + (1 << 20)     # the frames, or the floor's slots (aligned bounds)
    dst = torch.empty(dst_cap, dtype=torch.uint8, device=dev)
    stream = torch.cuda.current_stream().cuda_stream
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def gpu_ms(fn):
        ev0.record(); fn(); ev1.record(); ev1.synchronize()
        return ev0.elapsed_time(ev1)

    def dev_write(offs, lens, bs, flags):
        fo, fl = np.zeros(len(lens), dtype=np.uint64), np.zeros(len(lens), dtype=np.uint64)
        r = lib.b200lz4f_compress_dev(src.data_ptr(), offs.ctypes.data, lens.ctypes.data, len(lens), dst.data_ptr(), dst_cap,
                                      fo.ctypes.data, fl.ctypes.data, bs, flags, 0, stream)
        return r, fo, fl

    def emit(rec):
        print(json.dumps(rec), flush=True)
        if args.json:
            with open(args.json, "a") as f:
                f.write(json.dumps(rec) + "\n")

    emit({"card": card(), "GiB": total / (1 << 30)})
    rng = np.random.default_rng(args.seed)
    for name, sizes in splits(total, rng).items():
        lens = np.asarray(sizes, dtype=np.uint64)
        offs = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.uint64)
        nh = int(np.searchsorted(np.cumsum(lens), int(args.host_gib * (1 << 30)), side="right"))
        nh = max(nh, 1)
        for bs in (4, 7):
            B = 1 << (8 + 2 * bs)
            boff = np.concatenate([o + np.arange(0, max(int(n), 1), B, dtype=np.uint64) for o, n in zip(offs, lens) if n])
            blen = np.concatenate([np.minimum(B, n - np.arange(0, int(n), B, dtype=np.uint64)) for n in lens if n])
            cb = blen + blen // 255 + 16                                 # compress bound, slots of it rounded up to 16
            slot = (cb + 15) // 16 * 16
            t_soff = torch.from_numpy(boff.astype(np.int64)).to(dev)
            t_slen = torch.from_numpy(blen.astype(np.int32)).to(dev)
            t_coff = torch.from_numpy((np.cumsum(slot) - slot).astype(np.int64)).to(dev)
            t_ccap = torch.from_numpy(cb.astype(np.int32)).to(dev)
            t_clen = torch.zeros(len(blen), device=dev, dtype=torch.int32)
            assert int(slot.sum()) <= dst_cap

            def floor():
                L.batch.compress_fast_batch_dev(src, t_soff, t_slen, dst, t_coff, t_ccap, t_clen, B if B <= 65536 else 0)

            for flags in (0, 2, 1):
                rec = {"split": name, "frames": len(lens), "bsCode": bs, "flags": flags}
                r, _, _ = dev_write(offs, lens, bs, flags)
                if r < 0:
                    rec["dev"] = f"refused ({r})"
                    emit(rec)
                    continue
                rec["bytes_out"] = int(r)
                hoffs, hlens = offs[:nh], lens[:nh]
                if int(lens[0]) > args.host_gib * (1 << 30):             # one frame larger than the host leg: a frame of host-gib
                    hoffs, hlens = offs[:1], np.asarray([int(args.host_gib * (1 << 30))], dtype=np.uint64)
                hbytes = int(hlens.sum())
                pinned = torch.empty(hbytes, dtype=torch.uint8, pin_memory=True)
                hdst = np.empty(sum(lib.b200lz4f_compress_bound(int(n), bs) for n in hlens), dtype=np.uint8)
                hsrc = pinned.numpy()

                def host():
                    t = time.perf_counter()
                    pinned.copy_(src[int(hoffs[0]):int(hoffs[0]) + hbytes])
                    o, outs = 0, []
                    for a, n in zip(hoffs - hoffs[0], hlens):
                        w = lib.b200lz4f_compress_host(hsrc.ctypes.data + int(a), int(n), hdst.ctypes.data + o, len(hdst) - o, bs, flags)
                        assert w > 0, w
                        outs.append((o, int(w))); o += int(w)
                    return (time.perf_counter() - t) * 1e3, outs

                t_dev, t_floor, t_host = [], [], []
                for k in range(args.warmup + args.runs):
                    a = gpu_ms(lambda: dev_write(offs, lens, bs, flags))
                    b = gpu_ms(floor)
                    if k >= args.warmup:
                        t_dev.append(a); t_floor.append(b)
                for k in range(args.host_runs):
                    t_host.append(host()[0])
                    gpu_ms(lambda: dev_write(offs, lens, bs, flags))     # alternate with the device writer
                # digests on the host leg's frames: the device writer's and the host writer's
                _, hout = host()
                r2, fo, fl = dev_write(hoffs, hlens, bs, flags)
                torch.cuda.synchronize()
                got = dst[:int(r2)].cpu().numpy()
                rec["digest_dev"] = hashlib.sha256(got.tobytes()).hexdigest()[:16]
                rec["digest_host"] = hashlib.sha256(b"".join(hdst[o:o + w].tobytes() for o, w in hout)).hexdigest()[:16]
                md, mf, mh = float(np.median(t_dev)), float(np.median(t_floor)), float(np.median(t_host))
                gib = total / (1 << 30)
                rec.update({"dev_ms": round(md, 2), "floor_ms": round(mf, 2), "dev_GiBps": round(gib / md * 1e3, 1),
                            "floor_GiBps": round(gib / mf * 1e3, 1), "dev_over_floor": round(md / mf, 3),
                            "host_GiB": round(hbytes / (1 << 30), 3), "host_ms": round(mh, 1),
                            "host_GiBps": round(hbytes / (1 << 30) / mh * 1e3, 2)})
                emit(rec)
                del pinned, hdst


if __name__ == "__main__":
    sys.exit(main())
