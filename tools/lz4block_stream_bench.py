"""Incremental device LZ4Block writer and reader (b200lz4block_writer_write_dev, b200lz4block_reader_read_dev) against the
whole-stream device calls, on one GPU.

The data: RDG P=0.5 (the bench corpus) from a seeded 256 MiB host sample, tiled across --gib GiB of device memory with the
first 8 bytes of every 64 KiB perturbed so that blocks differ, cut into 1, 64 and 4096 streams at 64 KiB blocks and into 1
and 64 streams at 256 KiB blocks (above 64 KiB the fast compressor's one-warp long kernel writes the blocks).  Median of
--runs after a warm-up, each timed by a host clock around work that ends in a device synchronise:
  writer:  a  b200lz4block_writer_write_dev, --piece-mib MiB per call in total shared over the streams (whole blocks, at
              least one per stream), WRITE until a stream's last piece, which is a CLOSE; each stream grows in its own range
           b  b200lz4block_compress_dev on the whole streams
           c  the fast block compressor alone (b200lz4_compress_fast_batch_dev) over the same blocks, descriptors prepared
  reader:  a  b200lz4block_reader_read_dev over compress_dev's streams, --piece-mib MiB per call in total (at least one
              whole unit per stream), room exact: what the stream has left to decode
           b  b200lz4block_decompress_dev on the whole streams
           c  the fast block decoder alone (b200lz4_decompress_fast_batch_dev) over the floor compressor's blocks
Checks: the writer's streams must be byte for byte compress_dev's (every piece starts at the content's phase), and every
reader arm must give back the source.  Also: the fixed cost of a call (one stream: a CLOSE that writes only the end block,
and a read of that end block, median of 200), and with --long-gib one stream of that much content (one 256 MiB device piece
written again and again) piped call by call into the incremental reader, every piece compared with the source.
    python tools/lz4block_stream_bench.py [--gib 8] [--runs 3] [--piece-mib 64,256] [--cuts 65536:1,65536:64,...]
"""
import argparse
import ctypes
import json
import sys
import time

import _variant  # noqa: F401  (B200LZ4_TEST_SO: another build of the library)
import numpy as np

from frame_streams_bench import card

H = 21


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=8)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--seed", type=int, default=2)
    ap.add_argument("--cuts", default="65536:1,65536:64,65536:4096,262144:1,262144:64",
                    help="blockSize:streams pairs, comma separated")
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

    def u64(a):
        return np.ascontiguousarray(np.asarray(a, dtype=np.uint64))

    def writer_pass(out, w_off, lens, offs, piece, bs):
        """every stream written to its close, `piece` bytes per call shared over the streams -> (ok, calls, stream lengths)"""
        ns = len(lens)
        err = ctypes.c_int(0)
        h = lib.b200lz4block_writer_create(ns, bs, 0, ctypes.byref(err))
        per = max(piece // ns // bs, 1) * bs
        pos, done = np.zeros(ns, dtype=np.uint64), np.zeros(ns, dtype=np.uint64)
        st = np.zeros(ns, dtype=np.int32)
        used, prod, need = (np.zeros(ns, dtype=np.uint64) for _ in range(3))
        calls = 0
        while True:
            s_off = u64(offs + pos)
            s_len = u64(np.minimum(lens - pos, np.uint64(per)))
            op = np.ascontiguousarray(np.where(pos + s_len == lens, 2, 0).astype(np.uint8))
            d_off = u64(w_off + done)
            d_cap = u64(s_len + (s_len // np.uint64(bs) + np.uint64(2)) * np.uint64(H))
            rc = lib.b200lz4block_writer_write_dev(h, src.data_ptr(), s_off.ctypes.data, s_len.ctypes.data, op.ctypes.data,
                                                   out.data_ptr(), d_off.ctypes.data, d_cap.ctypes.data, st.ctypes.data,
                                                   used.ctypes.data, prod.ctypes.data, need.ctypes.data, stream)
            calls += 1
            if rc != 0 or (st == 1).any():
                lib.b200lz4block_writer_free(h)
                return False, calls, done
            pos += used
            done += prod
            if (st == 2).all():
                break
        lib.b200lz4block_writer_free(h)
        return bool((pos == lens).all()), calls, done

    def reader_pass(streams, so, sl, out, offs, lens, piece, bs, stop=1):
        """every stream read to DONE, `piece` bytes per call shared over the streams, room exact -> (ok, calls)"""
        ns = len(sl)
        err = ctypes.c_int(0)
        h = lib.b200lz4block_reader_create(ns, stop, ctypes.byref(err))
        per = np.uint64(max(piece // ns, bs + bs // 255 + 16 + H + H))
        pos, done = np.zeros(ns, dtype=np.uint64), np.zeros(ns, dtype=np.uint64)
        st = np.zeros(ns, dtype=np.int32)
        used, prod, need = (np.zeros(ns, dtype=np.uint64) for _ in range(3))
        calls = 0
        while True:
            s_off = u64(so + pos)
            s_len = u64(np.minimum(sl - pos, per))
            eof = np.ascontiguousarray((pos + s_len == sl).astype(np.uint8))
            d_off = u64(offs + done)
            d_cap = u64(lens - done)
            rc = lib.b200lz4block_reader_read_dev(h, streams.data_ptr(), s_off.ctypes.data, s_len.ctypes.data, eof.ctypes.data,
                                                  out.data_ptr(), d_off.ctypes.data, d_cap.ctypes.data, st.ctypes.data,
                                                  used.ctypes.data, prod.ctypes.data, need.ctypes.data, stream)
            calls += 1
            if rc != 0 or (st < 0).any() or (st == 1).any():
                lib.b200lz4block_reader_free(h)
                return False, calls
            pos += used
            done += prod
            if (st == 2).all():
                break
        lib.b200lz4block_reader_free(h)
        return bool((pos == sl).all() and (done == lens).all()), calls

    emit({"card": card(), "GiB": total / (1 << 30)})
    # the fixed cost of a call: one stream; a CLOSE that writes only the end block, then a read of that end block
    scratch = torch.zeros(1 << 20, dtype=torch.uint8, device=dev)
    z, room = np.zeros(1, dtype=np.uint64), np.full(1, 64, dtype=np.uint64)
    ln21 = np.full(1, H, dtype=np.uint64)
    one = np.ones(1, dtype=np.uint8)
    close = np.full(1, 2, dtype=np.uint8)
    st = np.zeros(1, dtype=np.int32)
    u, p_, nd = (np.zeros(1, dtype=np.uint64) for _ in range(3))
    tw, tr = [], []
    for k in range(220):
        err = ctypes.c_int(0)
        h = lib.b200lz4block_writer_create(1, BLK, 0, ctypes.byref(err))
        t, _ = clock(lambda: lib.b200lz4block_writer_write_dev(h, src.data_ptr(), z.ctypes.data, z.ctypes.data, close.ctypes.data,
                                                               scratch.data_ptr(), z.ctypes.data, room.ctypes.data, st.ctypes.data,
                                                               u.ctypes.data, p_.ctypes.data, nd.ctypes.data, stream))
        lib.b200lz4block_writer_free(h)
        assert int(st[0]) == 2 and int(p_[0]) == H
        if k >= 20:
            tw.append(t)
        h = lib.b200lz4block_reader_create(1, 1, ctypes.byref(err))
        t, _ = clock(lambda: lib.b200lz4block_reader_read_dev(h, scratch.data_ptr(), z.ctypes.data, ln21.ctypes.data, one.ctypes.data,
                                                              scratch.data_ptr(), room.ctypes.data, room.ctypes.data, st.ctypes.data,
                                                              u.ctypes.data, p_.ctypes.data, nd.ctypes.data, stream))
        lib.b200lz4block_reader_free(h)
        assert int(st[0]) == 2 and int(u[0]) == H
        if k >= 20:
            tr.append(t)
    emit({"fixed_cost_per_call_ms": {"writer": round(float(np.median(tw)), 3), "reader": round(float(np.median(tr)), 3)}})

    if args.long_gib:
        piece = src[:256 << 20]
        n = piece.numel()
        calls = (args.long_gib << 30) // n
        out = torch.empty(lib.b200lz4block_compress_bound(n, BLK) + 64, dtype=torch.uint8, device=dev)
        content = torch.empty(n, dtype=torch.uint8, device=dev)

        def run_long():
            good, produced = True, 0
            with L.LZ4BlockWriter(1, BLK) as wr, L.LZ4BlockReader(1) as rd:
                for c in range(calls + 1):
                    last = c == calls
                    s, used_, prod_, _ = wr.write(piece, [0], [0 if last else n], out, [0], [out.numel()], [2 if last else 0])
                    p = int(prod_[0])
                    rs, ru, rp, _ = rd.read(out, [0], [p], content, [0], [n], [last])
                    good &= int(ru[0]) == p and int(rs[0]) == (2 if last else 0)
                    if not last:
                        good &= int(rp[0]) == n and bool(torch.equal(content, piece))
                    produced += int(rp[0])
            return good and produced == calls * n
        t, good = clock(run_long)
        emit({"long_stream_GiB": args.long_gib, "piece_MiB": 256, "calls": calls + 1, "ok": good, "ms": round(t, 1),
              "GiBps_write_and_read": round(args.long_gib / t * 1e3, 2), "note": "includes a torch.equal of every piece"})

    pieces = [int(x) << 20 for x in args.piece_mib.split(",")]
    back = torch.empty(total + 64, dtype=torch.uint8, device=dev)
    for bs, ns in (tuple(int(y) for y in x.split(":")) for x in args.cuts.split(",")):
        lens = np.full(ns, total // ns // bs * bs, dtype=np.uint64)
        lens[-1] += total - int(lens.sum())
        offs = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.uint64)
        bounds = np.asarray([lib.b200lz4block_compress_bound(int(n), bs) for n in lens], dtype=np.uint64)
        cap = int(bounds.sum())
        streams = torch.empty(cap + 64, dtype=torch.uint8, device=dev)
        w_off = np.concatenate([[0], np.cumsum(bounds + np.uint64(64))[:-1]]).astype(np.uint64)
        so, sl = np.zeros(ns, dtype=np.uint64), np.zeros(ns, dtype=np.uint64)
        # the floors' blocks: every stream's, bound-sized slots in wout
        b_soff = np.concatenate([np.arange(int(o), int(o) + int(n), bs, dtype=np.uint64) for o, n in zip(offs, lens)])
        b_len = np.minimum(np.uint64(bs), np.concatenate([o + n - np.arange(int(o), int(o) + int(n), bs, dtype=np.uint64)
                                                          for o, n in zip(offs, lens)])).astype(np.int32)
        b_cap = (b_len + b_len // 255 + 16).astype(np.int32)
        slot = (b_cap.astype(np.uint64) + 15) // 16 * 16
        b_doff = (np.cumsum(slot) - slot).astype(np.uint64)
        wout = torch.empty(max(cap + ns * 64, int(slot.sum())) + 64, dtype=torch.uint8, device=dev)
        nblocks = len(b_soff)
        d_soff, d_len = torch.from_numpy(b_soff.view(np.int64)).to(dev), torch.from_numpy(b_len).to(dev)
        d_doff, d_cap = torch.from_numpy(b_doff.view(np.int64)).to(dev), torch.from_numpy(b_cap).to(dev)
        d_res = torch.empty(nblocks, dtype=torch.int32, device=dev)
        d_dres = torch.empty(nblocks, dtype=torch.int32, device=dev)
        res = np.zeros(ns, dtype=np.int64)
        mlong = 65536 if bs <= 65536 else 0

        def w_compress_dev():
            return lib.b200lz4block_compress_dev(src.data_ptr(), offs.ctypes.data, lens.ctypes.data, ns, streams.data_ptr(), cap,
                                                 so.ctypes.data, sl.ctypes.data, bs, 0, stream) > 0

        def w_floor():
            return lib.b200lz4_compress_fast_batch_dev(src.data_ptr(), d_soff.data_ptr(), d_len.data_ptr(), wout.data_ptr(),
                                                       d_doff.data_ptr(), d_cap.data_ptr(), d_res.data_ptr(), nblocks, mlong,
                                                       stream) == 0

        def r_decompress_dev():
            rc = lib.b200lz4block_decompress_dev(streams.data_ptr(), so.ctypes.data, sl.ctypes.data, ns, back.data_ptr(),
                                                 offs.ctypes.data, lens.ctypes.data, 1, res.ctypes.data, None, None, stream)
            return rc == 0 and bool((res == lens.astype(np.int64)).all())

        def r_floor():       # the floor compressor's blocks in wout, decoded by the fast decoder alone
            return lib.b200lz4_decompress_fast_batch_dev(wout.data_ptr(), d_doff.data_ptr(), d_res.data_ptr(), back.data_ptr(),
                                                         d_soff.data_ptr(), d_len.data_ptr(), d_dres.data_ptr(), nblocks,
                                                         stream) == 0

        calls, match = {}, {}
        # the writer: its streams in wout must be compress_dev's
        warms = {"b_compress_dev": w_compress_dev, "c_floor": w_floor}
        for p in pieces:
            def a_writer(p=p):
                ok, calls[f"writer_{p >> 20}MiB"], wl = writer_pass(wout, w_off, lens, offs, p, bs)
                match[f"a_writer_{p >> 20}MiB_len"] = bool((wl == sl).all()) if sl.any() else None
                return ok
            warms[f"a_writer_{p >> 20}MiB"] = a_writer
        times = {k: [] for k in warms}
        for k in range(args.warmup + args.runs):
            for name, fn in warms.items():
                t, r = clock(fn)
                assert r, ("writer", name, bs, ns)
                if k == 0 and name.startswith("a_writer"):
                    match[name] = all(torch.equal(wout[int(w):int(w) + int(n)], streams[int(o):int(o) + int(n)])
                                      for w, o, n in zip(w_off, so, sl))
                if k >= args.warmup:
                    times[name].append(t)
        gib = total / (1 << 30)
        rec = {"call": "writer", "blockSize": bs, "streams": ns, "blocks": nblocks, "match": match,
               "calls": {k: c for k, c in calls.items() if k.startswith("writer")}}
        for name in warms:
            m = float(np.median(times[name]))
            rec[name + "_ms"] = round(m, 2)
            rec[name + "_GiBps"] = round(gib / m * 1e3, 1)
        emit(rec)
        assert all(v is not False for v in match.values()), match

        # the reader: compress_dev's streams (still in `streams`) and the floor compressor's blocks (still in wout)
        w_compress_dev()
        w_floor()
        ok_floor = bool((d_res.cpu().numpy() > 0).all())
        rarms = {"b_decompress_dev": r_decompress_dev}
        if ok_floor:
            rarms["c_floor"] = r_floor
        for p in pieces:
            def a_reader(p=p):
                ok, calls[f"reader_{p >> 20}MiB"] = reader_pass(streams, so, sl, back, offs, lens, p, bs)
                return ok
            rarms[f"a_reader_{p >> 20}MiB"] = a_reader
        times = {k: [] for k in rarms}
        rmatch = {}
        for k in range(args.warmup + args.runs):
            for name, fn in rarms.items():
                back[:total].zero_()
                t, r = clock(fn)
                assert r, ("reader", name, bs, ns)
                if k == 0:
                    rmatch[name] = bool(torch.equal(back[:total], src))
                if k >= args.warmup:
                    times[name].append(t)
        rec = {"call": "reader", "blockSize": bs, "streams": ns, "blocks": nblocks, "match": rmatch,
               "calls": {k: c for k, c in calls.items() if k.startswith("reader")}}
        for name in rarms:
            m = float(np.median(times[name]))
            rec[name + "_ms"] = round(m, 2)
            rec[name + "_GiBps"] = round(gib / m * 1e3, 1)
        emit(rec)
        assert all(rmatch.values()), rmatch
        del streams, wout, d_soff, d_len, d_doff, d_cap, d_res, d_dres
        torch.cuda.empty_cache()


if __name__ == "__main__":
    sys.exit(main())
