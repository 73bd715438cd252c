"""Incremental device frame reader (b200lz4f_reader_read_dev) against the whole-stream device reader, on one GPU.

The data: RDG P=0.5 (the bench corpus) from a seeded 256 MiB host sample, tiled across --gib GiB of device memory with the
first 8 bytes of every 64 KiB perturbed so that blocks differ, written by b200lz4f_compress_dev with flags 0 and with flags 5
(content checksum and content size), cut into 1, 64 and 4096 streams at bsCode 4 and 7.  Three ways to read them, median of
--runs after a warm-up, each timed by a host clock around work that ends in a device synchronise:
  a  reader   b200lz4f_reader_read_dev, --piece-mib MiB per call in total shared over the streams, each stream's content
              packed straight into its place in the output
  b  streams  b200lz4f_decompress_streams_dev on the whole streams
  c  floor    the safe block decoder alone (b200lz4_decompress_safe_batch_dev) over the same blocks, descriptors prepared
Every arm's output is compared with the source on the device.  Also: the fixed cost of a call (one stream, a piece of one
frame header, median of 200), and with --long-gib one stream of that much content (one 4 MiB block repeated, bsCode 7,
content size declared) read in --long-piece-mib pieces.
    python tools/frame_reader_bench.py [--gib 8] [--runs 3] [--piece-mib 64,256] [--flags 0,5] [--cuts 4:1,4:64,4:4096,7:1,7:64]
"""
import argparse
import json
import sys
import time

import _variant  # noqa: F401  (B200LZ4_TEST_SO: another build of the library)
import numpy as np

from frame_streams_bench import blocks_of, card


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=8)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--seed", type=int, default=2)
    ap.add_argument("--flags", default="0,5")
    ap.add_argument("--cuts", default="4:1,4:64,4:4096,7:1,7:64,7:4096", help="bsCode:streams pairs, comma separated")
    ap.add_argument("--piece-mib", default="64,256", help="bytes per call in total, comma separated")
    ap.add_argument("--long-gib", type=int, default=0, help="also read one stream of this much content in pieces")
    ap.add_argument("--long-piece-mib", type=int, default=256)
    ap.add_argument("--json", default="")
    args = ap.parse_args()

    import torch
    import lz4java_b200 as L
    from oracle import oracle as O
    lib = L._native.lib()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    port = O.best_available()

    BLK = 65536
    total = int(args.gib * (1 << 30)) // BLK * BLK
    base_n = min(total, 256 << 20)
    base = torch.from_numpy(port.datagen(base_n, 0.5, 0.0, args.seed)).to(dev)
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
    out = torch.empty(total + (4 << 20) + 64, dtype=torch.uint8, device=dev)

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

    def reader_pass(frames, fo, fl, lens, offs, piece, bsz):
        """every stream read to its end, `piece` bytes per call shared over the streams -> (ok, calls)"""
        import ctypes
        ns = len(fl)
        err = ctypes.c_int(0)
        h = lib.b200lz4f_reader_create(ns, 0, ctypes.byref(err))
        pos = np.zeros(ns, dtype=np.uint64)
        done = np.zeros(ns, dtype=np.uint64)
        per = max(piece // ns, 16)
        st = np.zeros(ns, dtype=np.int32)
        used, prod, need = (np.zeros(ns, dtype=np.uint64) for _ in range(3))
        calls = 0
        while True:
            s_off = np.ascontiguousarray(fo + pos)
            s_len = np.ascontiguousarray(np.minimum(fl - pos, np.maximum(np.uint64(per), need)))   # at least the next unit
            eof = np.ascontiguousarray((pos + s_len == fl).astype(np.uint8))
            d_off = np.ascontiguousarray(offs + done)
            d_cap = np.ascontiguousarray(lens - done + np.uint64(bsz))
            rc = lib.b200lz4f_reader_read_dev(h, frames.data_ptr(), s_off.ctypes.data, s_len.ctypes.data, eof.ctypes.data,
                                              out.data_ptr(), d_off.ctypes.data, d_cap.ctypes.data, st.ctypes.data,
                                              used.ctypes.data, prod.ctypes.data, need.ctypes.data, stream)
            calls += 1
            if rc != 0 or (st < 0).any():
                lib.b200lz4f_reader_free(h)
                return False, calls
            pos += used
            done += prod
            if (st == 2).all():
                break
        lib.b200lz4f_reader_free(h)
        return bool((done == lens).all()), calls

    emit({"card": card(), "GiB": total / (1 << 30)})
    # the fixed cost of a call: one stream, a piece that holds only a frame header
    import ctypes
    hdr = torch.from_numpy(np.frombuffer(L.compress_frame(b"x" * 100, 4, True, False, False), dtype=np.uint8).copy()).to(dev)
    ts = []
    one = np.zeros(1, dtype=np.uint64)
    seven, no = np.full(1, 7, dtype=np.uint64), np.zeros(1, dtype=np.uint8)
    st = np.zeros(1, dtype=np.int32)
    u, p_, nd = (np.zeros(1, dtype=np.uint64) for _ in range(3))
    for k in range(220):
        err = ctypes.c_int(0)
        h = lib.b200lz4f_reader_create(1, 0, ctypes.byref(err))
        t, _ = clock(lambda: lib.b200lz4f_reader_read_dev(h, hdr.data_ptr(), one.ctypes.data, seven.ctypes.data, no.ctypes.data,
                                                          out.data_ptr(), one.ctypes.data, one.ctypes.data, st.ctypes.data,
                                                          u.ctypes.data, p_.ctypes.data, nd.ctypes.data, stream))
        lib.b200lz4f_reader_free(h)
        if k >= 20:
            ts.append(t)
    emit({"fixed_cost_per_call_ms": round(float(np.median(ts)), 3)})

    if args.long_gib:
        bs = 4 << 20
        content = port.datagen(bs, 0.5, 0.0, 17).tobytes()
        block = L.compress_frame(content, 7, False, False, False)[7:-4]
        d_content = torch.from_numpy(np.frombuffer(content, dtype=np.uint8).copy()).to(dev)
        per = (args.long_piece_mib << 20) // len(block)
        body = torch.from_numpy(np.frombuffer(block, dtype=np.uint8).copy()).to(dev).repeat(per)
        n = (args.long_gib << 30) // bs
        d = bytes([0x68, 0x70]) + (n * bs).to_bytes(8, "little")
        head = torch.from_numpy(np.frombuffer(b"\x04\x22\x4d\x18" + d + bytes([(port.xxh32(d, 0) >> 8) & 0xFF]), dtype=np.uint8).copy()).to(dev)
        last = n - per * ((n - 1) // per)                                  # blocks of the last piece
        tail = torch.cat([body[:last * len(block)], torch.zeros(4, dtype=torch.uint8, device=dev)])
        rd = L.FrameReader(1)
        dst = out[:per * bs]

        def run_long():
            left, good, calls = n, True, 1
            rd.read(head, [0], [head.numel()], dst, [0], [0], [False])
            while True:
                k = min(left, per)
                piece, eof = (body, False) if left > per else (tail, True)
                s, _, prod, _ = rd.read(piece, [0], [piece.numel()], dst, [0], [per * bs], [eof])
                calls += 1
                good &= int(prod[0]) == k * bs and bool((dst[:k * bs].view(k, bs) == d_content).all())
                left -= k
                if s[0] != 0:
                    return good and int(s[0]) == 2 and left == 0, calls
        t, (good, calls) = clock(run_long)
        rd.close()
        emit({"long_stream_GiB": args.long_gib, "piece_MiB": args.long_piece_mib, "calls": calls, "ok": good,
              "ms": round(t, 1), "GiBps_incl_check": round(args.long_gib / t * 1e3, 1)})

    pieces = [int(x) << 20 for x in args.piece_mib.split(",")]
    for flags in (int(x) for x in args.flags.split(",")):
        for bs, ns in (tuple(int(y) for y in x.split(":")) for x in args.cuts.split(",")):
            lens = np.full(ns, total // ns, dtype=np.uint64)
            lens[-1] += total - int(lens.sum())
            offs = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.uint64)
            frames, fo, fl = L.compress_frames_dev(src, offs, lens, block_size_code=bs, content_checksum=bool(flags & 1),
                                                   content_size=bool(flags & 4))
            torch.cuda.synchronize()
            fo, fl = np.ascontiguousarray(fo), np.ascontiguousarray(fl)
            bsz = 1 << (8 + 2 * bs)
            b_soff, b_size, b_raw, b_kin = blocks_of(frames.cpu().numpy(), fo)
            assert not b_raw.any(), "RDG P=0.5 blocks all shrink: the floor decodes compressed blocks only"
            nblocks = len(b_soff)
            frame_of = np.cumsum(b_kin == 0) - 1
            b_doff = offs[frame_of] + b_kin * np.uint64(bsz)
            b_cap = np.minimum(np.uint64(bsz), offs[frame_of] + lens[frame_of] - b_doff).astype(np.int32)
            d_soff, d_slen = torch.from_numpy(b_soff.view(np.int64)).to(dev), torch.from_numpy(b_size).to(dev)
            d_doff, d_cap = torch.from_numpy(b_doff.view(np.int64)).to(dev), torch.from_numpy(b_cap).to(dev)
            d_res = torch.empty(nblocks, dtype=torch.int32, device=dev)
            res = np.zeros(ns, dtype=np.int64)
            calls = {}

            def b_streams():
                rc = lib.b200lz4f_decompress_streams_dev(frames.data_ptr(), fo.ctypes.data, fl.ctypes.data, ns, out.data_ptr(),
                                                         offs.ctypes.data, lens.ctypes.data, 0, res.ctypes.data, None, None, stream)
                return rc == 0 and bool((res == lens.astype(np.int64)).all())

            def c_floor():
                return lib.b200lz4_decompress_safe_batch_dev(frames.data_ptr(), d_soff.data_ptr(), d_slen.data_ptr(), out.data_ptr(),
                                                             d_doff.data_ptr(), d_cap.data_ptr(), d_res.data_ptr(), nblocks, stream) == 0

            arms = {"b_streams": b_streams, "c_floor": c_floor}
            for p in pieces:
                def a_reader(p=p):
                    ok, calls[p] = reader_pass(frames, fo, fl, lens, offs, p, bsz)
                    return ok
                arms[f"a_reader_{p >> 20}MiB"] = a_reader
            times = {k: [] for k in arms}
            ok = {}
            for k in range(args.warmup + args.runs):
                for name, fn in arms.items():
                    if k == 0:
                        out.zero_()
                    t, r = clock(fn)
                    assert r, (name, flags, bs, ns)
                    if k == 0:
                        ok[name] = torch.equal(out[:total], src)
                    if k >= args.warmup:
                        times[name].append(t)
            rec = {"flags": flags, "bsCode": bs, "streams": ns, "blocks": nblocks, "match": ok,
                   "calls": {f"{p >> 20}MiB": c for p, c in calls.items()}}
            gib = total / (1 << 30)
            for name in arms:
                m = float(np.median(times[name]))
                rec[name + "_ms"] = round(m, 2)
                rec[name + "_GiBps"] = round(gib / m * 1e3, 1)
            emit(rec)
            del frames, d_soff, d_slen, d_doff, d_cap, d_res
            torch.cuda.empty_cache()

if __name__ == "__main__":
    sys.exit(main())
