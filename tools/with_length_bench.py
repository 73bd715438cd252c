"""Device WithLength writer and reader (b200lz4_compress_with_length_dev, b200lz4_decompress_with_length_dev) against their
floors, on one GPU.

The data: RDG P=0.5 (the bench corpus) from a seeded 256 MiB host sample, tiled across --gib GiB of device memory with the
first 8 bytes of every 4 KiB perturbed so that records differ, cut into records of 4 KiB, of 64 KiB, and of a seeded mix of
1 KiB to 256 KiB.  Median of --runs after a warm-up, each timed by a host clock around work that ends in a device
synchronise:
  writer        b200lz4_compress_with_length_dev over all records
  floor         b200lz4_compress_fast_batch_dev over the same records into bound-sized slots (the compressor alone; for the
                mix, one call per compressor class: records of up to 64 KiB with max_src_len 65536, the longer ones with 0)
  reader fast   b200lz4_decompress_with_length_dev, safe = 0, of the written records into a device buffer
  floor         b200lz4_decompress_fast_batch_dev over the same blocks
  reader safe   the same with safe = 1
  floor         b200lz4_decompress_safe_batch_dev over the same blocks
Every arm's output is checked: the records decode to the source, both readers and both floor decoders give the source back.
    python tools/with_length_bench.py [--gib 8] [--runs 3]
"""
import argparse
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=8)
    ap.add_argument("--runs", type=int, default=3)
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

    total = int(args.gib * (1 << 30)) // (1 << 20) * (1 << 20)
    base_n = min(total, 256 << 20)
    base = torch.from_numpy(O.best_available().datagen(base_n, 0.5, 0.0, args.seed)).to(dev)
    src = torch.empty(total + 64, dtype=torch.uint8, device=dev)
    for lo in range(0, total, base_n):
        src[lo:lo + base_n] = base[:min(base_n, total - lo)]
    src[total:] = 0
    nblk = total // 4096
    idx = torch.arange(nblk, device=dev, dtype=torch.int64)
    v = src[:total].view(nblk, 4096)
    for k in range(8):
        v[:, k] ^= ((idx >> (8 * k)) & 0xFF).to(torch.uint8)
    del base, idx, v
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

    def cuda_u64(a):
        return torch.from_numpy(np.ascontiguousarray(a, dtype=np.int64)).to(dev)

    def cuda_i32(a):
        return torch.from_numpy(np.ascontiguousarray(a, dtype=np.int32)).to(dev)

    emit({"card": card(), "GiB": total / (1 << 30)})
    gib = total / (1 << 30)
    rng = np.random.default_rng(args.seed)
    mix = rng.integers(1 << 10, (256 << 10) + 1, total // (128 << 10) * 2)
    mix = mix[:np.searchsorted(np.cumsum(mix), total)]
    mix = np.append(mix, total - int(mix.sum()))
    for name, lens in (("4KiB", np.full(total // 4096, 4096)), ("64KiB", np.full(total // 65536, 65536)), ("1-256KiB", mix)):
        lens = lens.astype(np.uint64)
        offs = (np.cumsum(lens) - lens).astype(np.uint64)
        n = len(lens)
        bound = int((lens + lens // 255 + 20).sum())
        recs = torch.empty(bound + 64, dtype=torch.uint8, device=dev)
        # the writer's floor: the compressor alone, per class, into bound-sized slots
        cap = (lens + lens // 255 + 16).astype(np.int64)
        slot = (cap + 15) // 16 * 16
        slots = torch.empty(int(slot.sum()) + 64, dtype=torch.uint8, device=dev)
        sl_off = np.cumsum(slot) - slot
        classes = []
        for wide in (True, False):
            sel = np.nonzero((lens <= 65536) == wide)[0]
            if len(sel):
                classes.append((cuda_u64(offs[sel]), cuda_i32(lens[sel]), cuda_u64(sl_off[sel]), cuda_i32(cap[sel]),
                                torch.zeros(len(sel), dtype=torch.int32, device=dev), 65536 if wide else 0))
        _, ro, rl = L.compress_with_length_dev(src, offs, lens, out=recs)
        b_soff, b_slen = cuda_u64(ro + 4), cuda_i32(rl - 4)
        d_off, d_len = cuda_u64(offs), cuda_i32(lens)
        b_res = torch.zeros(n, dtype=torch.int32, device=dev)
        t = {k: [] for k in ("writer", "writer_floor", "fast", "fast_floor", "safe", "safe_floor")}
        ok = {}

        def writer():
            return L.compress_with_length_dev(src, offs, lens, out=recs)

        def writer_floor():
            for a in classes:
                L.batch.compress_fast_batch_dev(src, a[0], a[1], slots, a[2], a[3], a[4], max_src_len=a[5])

        def reader(safe):
            return L.decompress_with_length_dev(recs, ro, rl, out, offs, lens, safe=safe)

        def reader_floor(safe):
            fn = L.batch.decompress_safe_batch_dev if safe else L.batch.decompress_fast_batch_dev
            fn(recs, b_soff, b_slen, out, d_off, d_len, b_res)

        for k in range(args.warmup + args.runs):
            tw, (_, ro2, rl2) = clock(writer)
            tfw, _ = clock(writer_floor)
            if k == 0:
                ok["writer"] = bool((ro2 == ro).all() and (rl2 == rl).all())
                ok["writer_floor"] = all(bool((a[4] > 0).all()) for a in classes)
            times = {"writer": tw, "writer_floor": tfw}
            for safe in (False, True):
                out.zero_()
                tr, (res, orig) = clock(lambda: reader(safe))
                if k == 0:
                    want = lens if safe else rl
                    ok["fast" if not safe else "safe"] = bool((res == want.astype(np.int64)).all() and
                                                              torch.equal(out[:total], src[:total]))
                out.zero_()
                tf, _ = clock(lambda: reader_floor(safe))
                if k == 0:
                    want = d_len if safe else b_slen
                    ok[("safe" if safe else "fast") + "_floor"] = bool(torch.equal(b_res, want) and torch.equal(out[:total], src[:total]))
                times["safe" if safe else "fast"], times[("safe" if safe else "fast") + "_floor"] = tr, tf
            if k >= args.warmup:
                for key, v in times.items():
                    t[key].append(v)
        med = {key: float(np.median(v)) for key, v in t.items()}
        rec = {"records": name, "n": n, "long_records": int((lens > 65536).sum()), "records_GiB": round(int(rl.sum()) / (1 << 30), 3),
               "match": ok}
        for key, m in med.items():
            rec[key + "_ms"] = round(m, 2)
            rec[key + "_GiBps"] = round(gib / m * 1e3, 1)
        rec["writer_over_floor"] = round(med["writer"] / med["writer_floor"], 3)
        rec["fast_over_floor"] = round(med["fast"] / med["fast_floor"], 3)
        rec["safe_over_floor"] = round(med["safe"] / med["safe_floor"], 3)
        emit(rec)
        del recs, slots, classes, b_soff, b_slen, d_off, d_len, b_res


if __name__ == "__main__":
    sys.exit(main())
