"""Device LZ4 Frame reader (b200lz4f_index_create_dev, b200lz4f_decompress_dev) against what a caller whose frames are in
device memory did without it, on one GPU.

The data: RDG P=0.5 (the bench corpus) from a seeded 256 MiB host sample, tiled across --gib GiB of device memory with the
first 8 bytes of every 64 KiB perturbed so that blocks differ, written by b200lz4f_compress_dev as bsCode 4 in 1, 64 and
4096 frames and bsCode 7 in 64 frames, flags 0 (a frame past 2 GiB cannot carry a content checksum).  Four ways to read them back, alternately in the same process,
median of --runs after a warm-up, each timed by a host clock around work that ends in a device synchronise:
  a  host    the container copied to pinned host memory, b200lz4f_index_create there, then b200lz4f_decode_dev
  b  dev     b200lz4f_index_create_dev without hints, then b200lz4f_decode_dev
  c  hints   the same with the writer's frame_off as hints
  d  e2e     b200lz4f_decompress_dev into a device buffer (index, decode into its scratch, pack)
The index alone is reported for a, b and c (a: the copy to the host and the host walk).  Every arm's decoded bytes are compared
with the source on the device, and the sha256 of the whole content is printed for arm d and for the source.
    python tools/frame_decode_bench.py [--gib 8] [--runs 5]
"""
import argparse
import ctypes
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


def sha(t, torch):
    h = hashlib.sha256()
    step = 1 << 30
    for lo in range(0, t.numel(), step):
        h.update(t[lo:lo + step].cpu().numpy().tobytes())
    return h.hexdigest()[:16]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=8)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
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
    src_sha = sha(src, torch)
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

    emit({"card": card(), "GiB": total / (1 << 30), "source_sha256": src_sha})
    for bs, nf in ((4, 1), (4, 64), (4, 4096), (7, 64)):
        lens = np.full(nf, total // nf, dtype=np.uint64)
        lens[-1] += total - int(lens.sum())
        offs = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.uint64)
        frames, fo, _ = L.compress_frames_dev(src, offs, lens, block_size_code=bs, content_checksum=False)
        torch.cuda.synchronize()
        n = frames.numel()
        hints = np.ascontiguousarray(fo)
        pinned = torch.empty(n, dtype=torch.uint8, pin_memory=True)
        slot = ctypes.c_uint64(0); err = ctypes.c_int(0)
        ix0 = lib.b200lz4f_index_create_dev(frames.data_ptr(), n, 0, None, 0, ctypes.byref(slot), None, ctypes.byref(err), stream)
        assert ix0 and err.value == 0, err.value
        nblocks = lib.b200lz4f_index_blocks(ix0)
        lib.b200lz4f_index_free(ix0)
        slots = torch.empty(slot.value + 64, dtype=torch.uint8, device=dev)
        foff, flen = np.zeros(nf, dtype=np.uint64), np.zeros(nf, dtype=np.uint64)

        def decode(ix):
            r = lib.b200lz4f_decode_dev(ix, frames.data_ptr(), slots.data_ptr(), foff.ctypes.data, flen.ctypes.data, None, stream)
            lib.b200lz4f_index_free(ix)
            return r

        def index_host():
            pinned.copy_(frames)
            torch.cuda.synchronize()
            return lib.b200lz4f_index_create(pinned.data_ptr(), n, ctypes.byref(slot), ctypes.byref(err))

        def index_dev(h):
            return lib.b200lz4f_index_create_dev(frames.data_ptr(), n, 0, h.ctypes.data if h is not None else None,
                                                 0 if h is None else len(h), ctypes.byref(slot), None, ctypes.byref(err), stream)

        def e2e():
            return lib.b200lz4f_decompress_dev(frames.data_ptr(), n, out.data_ptr(), total, 0, hints.ctypes.data, len(hints), None, stream)

        arms = {"a_host": lambda: index_host(), "b_dev": lambda: index_dev(None), "c_hints": lambda: index_dev(hints)}
        t_ix = {k: [] for k in arms}
        t_all = {k: [] for k in list(arms) + ["d_e2e"]}
        ok = {}
        for k in range(args.warmup + args.runs):
            for name, mk in arms.items():
                ti, ix = clock(mk)
                assert ix, (name, err.value)
                td, r = clock(lambda: decode(ix))
                assert r == total, (name, r)
                if k >= args.warmup:
                    t_ix[name].append(ti); t_all[name].append(ti + td)
                if k == 0:
                    ok[name] = all(torch.equal(slots[int(o):int(o) + int(m)], src[int(a):int(a) + int(m)])
                                   for o, m, a in zip(foff, flen, offs))
            te, r = clock(e2e)
            assert r == total, ("d_e2e", r)
            if k >= args.warmup:
                t_all["d_e2e"].append(te)
        ok["d_e2e"] = torch.equal(out[:total], src)
        rec = {"bsCode": bs, "frames": nf, "blocks": int(nblocks), "container_GiB": round(n / (1 << 30), 3),
               "content_sha256_e2e": sha(out[:total], torch), "match": ok}
        gib = total / (1 << 30)
        for name in t_all:
            m = float(np.median(t_all[name]))
            rec[name + "_ms"] = round(m, 2)
            rec[name + "_GiBps"] = round(gib / m * 1e3, 1)
            if name in t_ix:
                rec[name + "_index_ms"] = round(float(np.median(t_ix[name])), 2)
        emit(rec)
        del pinned, slots, frames


if __name__ == "__main__":
    sys.exit(main())
