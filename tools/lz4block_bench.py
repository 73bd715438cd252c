"""Device LZ4Block writer and reader (b200lz4block_compress_dev, b200lz4block_decompress_dev) against their floors and against
what a caller whose streams are in device memory does without them, on one GPU.

The data: RDG P=0.5 (the bench corpus) from a seeded 256 MiB host sample, tiled across --gib GiB of device memory with the
first 8 bytes of every 32 KiB perturbed so that blocks differ, cut into 1, 64 and 4096 streams of equal length, at block
sizes of 32 KiB and 64 KiB.  Median of --runs after a warm-up, each timed by a host clock around work that ends in a device
synchronise:
  a  writer      b200lz4block_compress_dev over all streams
     floor       b200lz4_compress_fast_batch_dev over the same blocks into bound-sized slots (the compressor alone)
  b  reader      b200lz4block_decompress_dev of the written streams into a device buffer
     floor       b200lz4_decompress_fast_batch_dev over the same compressed blocks (stored blocks are not decoded by it)
  c  host path   each stream copied to pinned host memory, b200lz4block_decompress_host, the content copied back
Every arm's output is checked against the source on the device.
    python tools/lz4block_bench.py [--gib 8] [--runs 3]
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


def blocks_of(host, so, sl):
    """(payload offset, compressed length, original length, raw) of every block of the streams, walked on the host copy"""
    out = []
    for o, n in zip(so.tolist(), sl.tolist()):
        ip, end = o, o + n
        while end - ip >= 21:
            clen = int.from_bytes(host[ip + 9:ip + 13].tobytes(), "little")
            olen = int.from_bytes(host[ip + 13:ip + 17].tobytes(), "little")
            raw = host[ip + 8] & 0xF0 == 0x10
            ip += 21
            if olen == 0:
                break
            out.append((ip, clen, olen, raw))
            ip += clen
    return out


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

    UNIT = 1 << 16
    total = int(args.gib * (1 << 30)) // (4096 * UNIT) * (4096 * UNIT)
    base_n = min(total, 256 << 20)
    base = torch.from_numpy(O.best_available().datagen(base_n, 0.5, 0.0, args.seed)).to(dev)
    src = torch.empty(total + 64, dtype=torch.uint8, device=dev)
    for lo in range(0, total, base_n):
        src[lo:lo + base_n] = base[:min(base_n, total - lo)]
    src[total:] = 0
    nblk = total // 32768
    idx = torch.arange(nblk, device=dev, dtype=torch.int64)
    v = src[:total].view(nblk, 32768)
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

    def cuda_u64(a):
        return torch.from_numpy(np.ascontiguousarray(a, dtype=np.int64)).to(dev)

    def cuda_i32(a):
        return torch.from_numpy(np.ascontiguousarray(a, dtype=np.int32)).to(dev)

    bound = lib.b200lz4block_compress_bound(total, 32768) + 4096 * 21
    pin_in = torch.empty(bound, dtype=torch.uint8, pin_memory=True)
    pin_out = torch.empty(total, dtype=torch.uint8, pin_memory=True)
    emit({"card": card(), "GiB": total / (1 << 30)})
    gib = total / (1 << 30)
    for bs in (32768, 65536):
        # the floor of the writer: the same blocks into bound-sized slots
        boff = np.arange(0, total, bs, dtype=np.uint64)
        blen = np.full(len(boff), bs, dtype=np.int32)
        bcap = blen + blen // 255 + 16
        bslot = np.cumsum((bcap.astype(np.uint64) + 15) // 16 * 16) - (bcap.astype(np.uint64) + 15) // 16 * 16
        slots = torch.empty(int(bslot[-1]) + int(bcap[-1]) + 64, dtype=torch.uint8, device=dev)
        f_off, f_len, f_slot, f_cap = cuda_u64(boff), cuda_i32(blen), cuda_u64(bslot), cuda_i32(bcap)
        f_res = torch.zeros(len(boff), dtype=torch.int32, device=dev)
        for ns in (1, 64, 4096):
            lens = np.full(ns, total // ns, dtype=np.uint64)
            offs = (np.arange(ns, dtype=np.uint64) * np.uint64(total // ns)).astype(np.uint64)
            t_w, t_fw, t_r, t_fr, t_h = [], [], [], [], []
            wbuf = torch.empty(sum(lib.b200lz4block_compress_bound(int(n), bs) for n in lens) + 64, dtype=torch.uint8, device=dev)
            streams, so, sl = L.compress_lz4block_dev(src, offs, lens, block_size=bs, out=wbuf)
            torch.cuda.synchronize()
            host = streams.cpu().numpy()
            blks = blocks_of(host, so, sl)
            comp = [b for b in blks if not b[3]]
            c_soff, c_slen = cuda_u64([b[0] for b in comp]), cuda_i32([b[1] for b in comp])
            dpos = np.cumsum([b[2] for b in blks]) - np.asarray([b[2] for b in blks])
            c_doff = cuda_u64([d for d, b in zip(dpos, blks) if not b[3]])
            c_dlen = cuda_i32([b[2] for b in comp])
            c_res = torch.zeros(len(comp), dtype=torch.int32, device=dev)
            ok = {}

            def writer():
                return L.compress_lz4block_dev(src, offs, lens, block_size=bs, out=wbuf)

            def writer_floor():
                L.batch.compress_fast_batch_dev(src, f_off, f_len, slots, f_slot, f_cap, f_res, max_src_len=65536)

            def reader():
                return L.decompress_lz4block_dev(streams, so, sl, out, offs, lens)

            def reader_floor():
                L.batch.decompress_fast_batch_dev(streams, c_soff, c_slen, out, c_doff, c_dlen, c_res)

            def host_path():
                pin_in[:streams.numel()].copy_(streams)
                rs = []
                for k in range(ns):
                    a, n = int(so[k]), int(sl[k])
                    rs.append(lib.b200lz4block_decompress_host(pin_in.data_ptr() + a, n, pin_out.data_ptr() + int(offs[k]),
                                                               int(lens[k]), 1, None))
                out[:total].copy_(pin_out)
                return rs

            for k in range(args.warmup + args.runs):
                tw, (got, so2, sl2) = clock(writer)
                tfw, _ = clock(writer_floor)
                tr, (res, _, _) = clock(reader)
                if k == 0:
                    ok["writer"] = bool((so2 == so).all() and (sl2 == sl).all())
                    ok["reader"] = bool((res == lens.astype(np.int64)).all() and torch.equal(out[:total], src[:total]))
                tfr, _ = clock(reader_floor)
                if k == 0:
                    ok["reader_floor"] = bool((c_res.cpu().numpy() == c_slen.cpu().numpy()).all())
                out.zero_()
                th, rs = clock(host_path)
                if k == 0:
                    ok["host"] = rs == [int(n) for n in lens] and torch.equal(out[:total], src[:total])
                if k >= args.warmup:
                    t_w.append(tw); t_fw.append(tfw); t_r.append(tr); t_fr.append(tfr); t_h.append(th)
            ok["writer_floor"] = bool((f_res.cpu().numpy() > 0).all())
            med = {n: float(np.median(t)) for n, t in (("a_writer", t_w), ("a_floor", t_fw), ("b_reader", t_r),
                                                        ("b_floor", t_fr), ("c_host", t_h))}
            rec = {"block_size": bs, "streams": ns, "blocks": len(blks), "stored_blocks": len(blks) - len(comp),
                   "streams_GiB": round(streams.numel() / (1 << 30), 3), "match": ok}
            for n, m in med.items():
                rec[n + "_ms"] = round(m, 2)
                rec[n + "_GiBps"] = round(gib / m * 1e3, 1)
            rec["writer_over_floor"] = round(med["a_writer"] / med["a_floor"], 3)
            rec["reader_over_floor"] = round(med["b_reader"] / med["b_floor"], 3)
            emit(rec)
            del streams, wbuf, c_soff, c_slen, c_doff, c_dlen, c_res
        del slots, f_off, f_len, f_slot, f_cap, f_res


if __name__ == "__main__":
    sys.exit(main())
