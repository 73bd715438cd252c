"""Incremental device frame writer (b200lz4f_writer_write_dev) against the whole-frame device writer, on one GPU.

The data: RDG P=0.5 (the bench corpus) from a seeded 256 MiB host sample, tiled across --gib GiB of device memory with the
first 8 bytes of every 64 KiB perturbed so that blocks differ, cut into 1, 64 and 4096 streams at bsCode 4 and 7, written with
flags 0 and with flags 5 (content checksum and content size).  Three ways to write them, median of --runs after a warm-up,
each timed by a host clock around work that ends in a device synchronise:
  a  writer       b200lz4f_writer_write_dev, --piece-mib MiB per call in total shared over the streams (at least one block
                  per stream), WRITE until a stream's last piece, which is a CLOSE; each stream's frame grows in its own range
  b  compress_dev b200lz4f_compress_dev on the whole frames
  c  floor        the fast block compressor alone (b200lz4_compress_fast_batch_dev) over the same blocks, descriptors prepared
The writer's frames must be byte for byte compress_dev's (every piece starts at the content's phase), and compress_dev's frames
are read back to the source by b200lz4f_decompress_streams_dev.  Also: the fixed cost of a call (one stream, a call that
writes only the header, median of 200), and with --long-gib one stream of that much content (one 256 MiB device piece
written again and again, bsCode 4, content size declared) piped call by call into the incremental reader.
    python tools/frame_writer_bench.py [--gib 8] [--runs 3] [--piece-mib 64,256] [--flags 0,5] [--cuts 4:1,4:64,4:4096,7:1,7:64]
"""
import argparse
import ctypes
import json
import sys
import time

import _variant  # noqa: F401  (B200LZ4_TEST_SO: another build of the library)
import numpy as np

from frame_streams_bench import card


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=8)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--seed", type=int, default=2)
    ap.add_argument("--flags", default="0,5")
    ap.add_argument("--cuts", default="4:1,4:64,4:4096,7:1,7:64,7:4096", help="bsCode:streams pairs, comma separated")
    ap.add_argument("--piece-mib", default="64,256", help="bytes per call in total, comma separated")
    ap.add_argument("--long-gib", type=int, default=0, help="also write one stream of this much content, piped into the reader")
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

    def writer_pass(out, w_off, lens, offs, piece, bs, flags, known):
        """every stream written to its close, `piece` bytes per call shared over the streams -> (ok, calls, frame lengths)"""
        ns = len(lens)
        bsz = 1 << (8 + 2 * bs)
        err = ctypes.c_int(0)
        h = lib.b200lz4f_writer_create(ns, bs, flags, 0, known.ctypes.data if flags & 4 else None, ctypes.byref(err))
        per = max(piece // ns // bsz, 1) * bsz
        pos = np.zeros(ns, dtype=np.uint64)
        done = np.zeros(ns, dtype=np.uint64)
        st = np.zeros(ns, dtype=np.int32)
        used, prod, need = (np.zeros(ns, dtype=np.uint64) for _ in range(3))
        calls = 0
        while True:
            s_off = np.ascontiguousarray(offs + pos)
            s_len = np.ascontiguousarray(np.minimum(lens - pos, np.uint64(per)))
            op = np.ascontiguousarray(np.where(pos + s_len == lens, 2, 0).astype(np.uint8))
            d_off = np.ascontiguousarray(w_off + done)
            d_cap = np.ascontiguousarray(s_len + (s_len // np.uint64(bsz) + np.uint64(1)) * np.uint64(8) + np.uint64(32))
            rc = lib.b200lz4f_writer_write_dev(h, src.data_ptr(), s_off.ctypes.data, s_len.ctypes.data, op.ctypes.data,
                                               out.data_ptr(), d_off.ctypes.data, d_cap.ctypes.data, st.ctypes.data,
                                               used.ctypes.data, prod.ctypes.data, need.ctypes.data, stream)
            calls += 1
            if rc != 0 or (st == 1).any():
                lib.b200lz4f_writer_free(h)
                return False, calls, done
            pos += used
            done += prod
            if (st == 2).all():
                break
        lib.b200lz4f_writer_free(h)
        return bool((pos == lens).all()), calls, done

    emit({"card": card(), "GiB": total / (1 << 30)})
    # the fixed cost of a call: one stream, a call that writes only the header
    scratch = torch.empty(1 << 20, dtype=torch.uint8, device=dev)
    ts = []
    z, room = np.zeros(1, dtype=np.uint64), np.full(1, 64, dtype=np.uint64)
    wop = np.zeros(1, dtype=np.uint8)
    st = np.zeros(1, dtype=np.int32)
    u, p_, nd = (np.zeros(1, dtype=np.uint64) for _ in range(3))
    for k in range(220):
        err = ctypes.c_int(0)
        h = lib.b200lz4f_writer_create(1, 4, 1, 0, None, ctypes.byref(err))
        t, _ = clock(lambda: lib.b200lz4f_writer_write_dev(h, src.data_ptr(), z.ctypes.data, z.ctypes.data, wop.ctypes.data,
                                                           scratch.data_ptr(), z.ctypes.data, room.ctypes.data, st.ctypes.data,
                                                           u.ctypes.data, p_.ctypes.data, nd.ctypes.data, stream))
        lib.b200lz4f_writer_free(h)
        if k >= 20:
            ts.append(t)
    emit({"fixed_cost_per_call_ms": round(float(np.median(ts)), 3)})

    if args.long_gib:
        piece = src[:256 << 20]
        n = piece.numel()
        calls = (args.long_gib << 30) // n
        out = torch.empty(n + (n >> 16) * 8 + 64, dtype=torch.uint8, device=dev)
        content = torch.empty(n, dtype=torch.uint8, device=dev)

        def run_long():
            wr = L.FrameWriter(1, 4, content_checksum=False, known_size=calls * n)
            rd = L.FrameReader(1, read_single_frame=True)
            good, produced = True, 0
            for c in range(calls + 1):
                close = c == calls
                s, used_, prod_, _ = wr.write(piece, [0], [0 if close else n], out, [0], [out.numel()], [2 if close else 0])
                p = int(prod_[0])
                rs, ru, rp, _ = rd.read(out, [0], [p], content, [0], [n], [close])
                good &= int(ru[0]) == p and int(rs[0]) == (2 if close else 0)
                produced += int(rp[0])
            wr.close()
            rd.close()
            return good and produced == calls * n and bool(torch.equal(content, piece))
        t, good = clock(run_long)
        emit({"long_stream_GiB": args.long_gib, "piece_MiB": 256, "calls": calls + 1, "ok": good, "ms": round(t, 1),
              "GiBps_write_and_read": round(args.long_gib / t * 1e3, 2)})

    pieces = [int(x) << 20 for x in args.piece_mib.split(",")]
    for flags in (int(x) for x in args.flags.split(",")):
        for bs, ns in (tuple(int(y) for y in x.split(":")) for x in args.cuts.split(",")):
            bsz = 1 << (8 + 2 * bs)
            lens = np.full(ns, total // ns, dtype=np.uint64)
            lens[-1] += total - int(lens.sum())
            offs = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.uint64)
            known = np.ascontiguousarray(lens.astype(np.int64))
            bounds = np.asarray([lib.b200lz4f_compress_bound(int(n), bs) for n in lens], dtype=np.uint64)
            cap = int(bounds.sum())
            frames = torch.empty(cap + 64, dtype=torch.uint8, device=dev)
            w_off = np.concatenate([[0], np.cumsum(bounds + np.uint64(64))[:-1]]).astype(np.uint64)
            fo, fl = np.zeros(ns, dtype=np.uint64), np.zeros(ns, dtype=np.uint64)
            # the floor's blocks: every stream's, bound-sized slots in wout
            b_soff = np.concatenate([np.arange(int(o), int(o) + int(n), bsz, dtype=np.uint64) for o, n in zip(offs, lens)])
            b_len = np.minimum(np.uint64(bsz), np.concatenate([o + n - np.arange(int(o), int(o) + int(n), bsz, dtype=np.uint64)
                                                               for o, n in zip(offs, lens)])).astype(np.int32)
            b_cap = (b_len + b_len // 255 + 16).astype(np.int32)
            slot = (b_cap.astype(np.uint64) + 15) // 16 * 16
            b_doff = (np.cumsum(slot) - slot).astype(np.uint64)
            wout = torch.empty(max(cap + ns * 64, int(slot.sum())) + 64, dtype=torch.uint8, device=dev)
            nblocks = len(b_soff)
            d_soff, d_len = torch.from_numpy(b_soff.view(np.int64)).to(dev), torch.from_numpy(b_len).to(dev)
            d_doff, d_cap = torch.from_numpy(b_doff.view(np.int64)).to(dev), torch.from_numpy(b_cap).to(dev)
            d_res = torch.empty(nblocks, dtype=torch.int32, device=dev)
            calls = {}

            def b_compress_dev():
                return lib.b200lz4f_compress_dev(src.data_ptr(), offs.ctypes.data, lens.ctypes.data, ns, frames.data_ptr(), cap,
                                                 fo.ctypes.data, fl.ctypes.data, bs, flags, 0, stream) > 0

            def c_floor():
                return lib.b200lz4_compress_fast_batch_dev(src.data_ptr(), d_soff.data_ptr(), d_len.data_ptr(), wout.data_ptr(),
                                                           d_doff.data_ptr(), d_cap.data_ptr(), d_res.data_ptr(), nblocks,
                                                           65536 if bsz <= 65536 else 0, stream) == 0

            # compress_dev refuses a content checksum over more than 0x7FFFFFFF bytes (-10): no baseline there
            refused = bool(flags & 1) and int(lens.max()) > 0x7FFFFFFF
            arms = {} if refused else {"b_compress_dev": b_compress_dev}
            arms["c_floor"] = c_floor
            wlen = {}
            for p in pieces:
                def a_writer(p=p):
                    ok, calls[p], wlen[p] = writer_pass(wout, w_off, lens, offs, p, bs, flags, known)
                    return ok
                arms[f"a_writer_{p >> 20}MiB"] = a_writer
            times = {k: [] for k in arms}
            match = {}
            for k in range(args.warmup + args.runs):
                for name, fn in arms.items():
                    t, r = clock(fn)
                    assert r, (name, flags, bs, ns)
                    if k == 0 and name.startswith("a_writer") and not refused:   # the writer's frames are compress_dev's
                        match[name] = all(torch.equal(wout[int(w):int(w) + int(n)], frames[int(o):int(o) + int(n)])
                                          for w, o, n in zip(w_off, fo, fl))
                    if k >= args.warmup:
                        times[name].append(t)
            # the last writer arm's frames (still in wout) read back to the source, content checksums checked
            back = torch.empty(total + 64, dtype=torch.uint8, device=dev)
            res = np.zeros(ns, dtype=np.int64)
            wl = np.ascontiguousarray(wlen[pieces[-1]])
            rc = lib.b200lz4f_decompress_streams_dev(wout.data_ptr(), w_off.ctypes.data, wl.ctypes.data, ns, back.data_ptr(),
                                                     offs.ctypes.data, lens.ctypes.data, 0, res.ctypes.data, None, None, stream)
            match["read_back"] = rc == 0 and bool((res == lens.astype(np.int64)).all()) and bool(torch.equal(back[:total], src))
            del back
            rec = {"flags": flags, "bsCode": bs, "streams": ns, "blocks": nblocks, "match": match,
                   "compress_dev": "refused (-10)" if refused else "ok",
                   "calls": {f"{p >> 20}MiB": c for p, c in calls.items()}}
            gib = total / (1 << 30)
            for name in arms:
                m = float(np.median(times[name]))
                rec[name + "_ms"] = round(m, 2)
                rec[name + "_GiBps"] = round(gib / m * 1e3, 1)
            emit(rec)
            del frames, wout, d_soff, d_len, d_doff, d_cap, d_res
            torch.cuda.empty_cache()


if __name__ == "__main__":
    sys.exit(main())
