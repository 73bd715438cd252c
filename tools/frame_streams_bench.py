"""Device reader of many LZ4 frame streams (b200lz4f_decompress_streams_dev) against what a caller whose frames are in device
memory has without it, on one GPU.

The data: RDG P=0.5 (the bench corpus) from a seeded 256 MiB host sample, tiled across --gib GiB of device memory with the
first 8 bytes of every 64 KiB perturbed so that blocks differ, written by b200lz4f_compress_dev with flags 0 and with flags 5
(content checksum and content size), cut into 64, 4096 and 65536 frames at bsCode 4 and 64 frames at bsCode 7.  Four ways to
read the frames back, alternately in the same process, median of --runs after a warm-up, each timed by a host clock around
work that ends in a device synchronise:
  a  streams  b200lz4f_decompress_streams_dev, one stream per frame, each into its own range of the output
  b  per      one b200lz4f_decompress_dev per frame (what a caller with frames scattered through a buffer had)
  c  concat   b200lz4f_decompress_dev on the frames back to back, the writer's frame_off as hints
  d  floor    the safe block decoder alone (b200lz4_decompress_safe_batch_dev) over the same blocks, descriptors prepared
Every arm's output is compared with the source on the device.  One more run of arm a under torch.profiler gives the device
time of each kernel it launches (a_kernels_ms), to show where the time goes.
(torch.profiler does not always return the kernels of a second profile in one process: the field is then empty.)
    python tools/frame_streams_bench.py [--gib 8] [--runs 3] [--flags 0,5] [--cuts 4:64,4:4096,4:65536,7:64]
"""
import argparse
import json
import struct
import subprocess
import sys
import time

import _variant  # noqa: F401  (B200LZ4_TEST_SO: another build of the library)
import numpy as np


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def blocks_of(h, fo):
    """the blocks of every frame of the container h (host bytes), walked in Python: (src_off, size, stored, block index in
    its frame) in frame order"""
    soff, size, raw, kin = [], [], [], []
    for f0 in fo:
        p = int(f0) + 4
        flg = int(h[p]); p += 2 + (8 if flg & 8 else 0) + 1
        k = 0
        while True:
            w = struct.unpack_from("<I", h, p)[0]; p += 4
            if w & 0x7FFFFFFF == 0:
                break
            soff.append(p); size.append(w & 0x7FFFFFFF); raw.append(w >> 31); kin.append(k)
            p += (w & 0x7FFFFFFF) + (4 if flg & 0x10 else 0); k += 1
    return np.array(soff, dtype=np.uint64), np.array(size, dtype=np.int32), np.array(raw, dtype=bool), np.array(kin, dtype=np.uint64)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=8)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--seed", type=int, default=2)
    ap.add_argument("--flags", default="0,5", help="frame flags to measure, comma separated")
    ap.add_argument("--cuts", default="4:64,4:4096,4:65536,7:64", help="bsCode:frames pairs to measure, comma separated")
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
    stream = torch.cuda.current_stream().cuda_stream
    out = torch.empty(total + 64, dtype=torch.uint8, device=dev)

    def emit(rec):
        print(json.dumps(rec), flush=True)
        if args.json:
            with open(args.json, "a") as f:
                f.write(json.dumps(rec) + "\n")

    def clock(fn):
        torch.cuda.synchronize()
        t = time.perf_counter()
        r = fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t) * 1e3, r

    emit({"card": card(), "GiB": total / (1 << 30)})
    for flags in (int(x) for x in args.flags.split(",")):
        for bs, nf in (tuple(int(y) for y in x.split(":")) for x in args.cuts.split(",")):
            lens = np.full(nf, total // nf, dtype=np.uint64)
            lens[-1] += total - int(lens.sum())
            offs = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.uint64)
            frames, fo, fl = L.compress_frames_dev(src, offs, lens, block_size_code=bs, content_checksum=bool(flags & 1),
                                                   content_size=bool(flags & 4))
            torch.cuda.synchronize()
            n = frames.numel()
            fo, fl = np.ascontiguousarray(fo), np.ascontiguousarray(fl)
            bsz = 1 << (8 + 2 * bs)
            # the floor's descriptors: every block, where its content goes (its frame's source offset + bs per block before it)
            b_soff, b_size, b_raw, b_kin = blocks_of(frames.cpu().numpy(), fo)
            assert not b_raw.any(), "RDG P=0.5 blocks all shrink: the floor decodes compressed blocks only"
            nblocks = len(b_soff)
            frame_of = np.cumsum(b_kin == 0) - 1                        # every frame has blocks
            b_doff = offs[frame_of] + b_kin * np.uint64(bsz)
            b_cap = np.minimum(np.uint64(bsz), offs[frame_of] + lens[frame_of] - b_doff).astype(np.int32)
            d_soff, d_slen = torch.from_numpy(b_soff.view(np.int64)).to(dev), torch.from_numpy(b_size).to(dev)
            d_doff, d_cap = torch.from_numpy(b_doff.view(np.int64)).to(dev), torch.from_numpy(b_cap).to(dev)
            d_res = torch.empty(nblocks, dtype=torch.int32, device=dev)
            res = np.zeros(nf, dtype=np.int64)

            def a_streams():
                rc = lib.b200lz4f_decompress_streams_dev(frames.data_ptr(), fo.ctypes.data, fl.ctypes.data, nf, out.data_ptr(),
                                                         offs.ctypes.data, lens.ctypes.data, 0, res.ctypes.data, None, None, stream)
                return rc == 0 and bool((res == lens.astype(np.int64)).all())

            def b_per():
                ok = True
                for f in range(nf):
                    r = lib.b200lz4f_decompress_dev(frames.data_ptr() + int(fo[f]), int(fl[f]), out.data_ptr() + int(offs[f]),
                                                    int(lens[f]), 0, None, 0, None, stream)
                    ok &= r == int(lens[f])
                return ok

            def c_concat():
                return lib.b200lz4f_decompress_dev(frames.data_ptr(), n, out.data_ptr(), total, 0, fo.ctypes.data, nf, None, stream) == total

            def d_floor():
                rc = lib.b200lz4_decompress_safe_batch_dev(frames.data_ptr(), d_soff.data_ptr(), d_slen.data_ptr(), out.data_ptr(),
                                                           d_doff.data_ptr(), d_cap.data_ptr(), d_res.data_ptr(), nblocks, stream)
                return rc == 0

            arms = {"a_streams": a_streams, "b_per_frame": b_per, "c_concat_hints": c_concat, "d_floor": d_floor}
            times = {k: [] for k in arms}
            ok = {}
            for k in range(args.warmup + args.runs):
                for name, fn in arms.items():
                    if k == 0:
                        out.zero_()
                    t, r = clock(fn)
                    assert r, (name, flags, bs, nf)
                    if k == 0:
                        if name == "d_floor":
                            assert bool((d_res == d_cap).all()), name
                        ok[name] = torch.equal(out[:total], src)
                    if k >= args.warmup:
                        times[name].append(t)
            rec = {"flags": flags, "bsCode": bs, "frames": nf, "blocks": nblocks, "container_GiB": round(n / (1 << 30), 3), "match": ok}
            gib = total / (1 << 30)
            for name in arms:
                m = float(np.median(times[name]))
                rec[name + "_ms"] = round(m, 2)
                rec[name + "_GiBps"] = round(gib / m * 1e3, 1)
            # where arm a's device time goes: one more run under the profiler, device time per kernel
            from torch.profiler import ProfilerActivity, profile
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                a_streams()
                torch.cuda.synchronize()
            per = {}
            for e in prof.events():
                if e.device_type.name == "CUDA":
                    key = e.name.split("(")[0].split("<")[0].replace("void ", "").replace("b200::", "")
                    per[key] = per.get(key, 0.0) + e.device_time_total / 1e3
            rec["a_kernels_ms"] = {k: round(t, 2) for k, t in sorted(per.items(), key=lambda kv: -kv[1]) if t >= 0.01}
            emit(rec)
            del frames, d_soff, d_slen, d_doff, d_cap, d_res
            torch.cuda.empty_cache()


if __name__ == "__main__":
    sys.exit(main())
