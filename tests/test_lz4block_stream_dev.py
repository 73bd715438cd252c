"""b200lz4block_writer_* / b200lz4block_reader_*: LZ4Block streams written and read in device memory piece by piece.  Each
writer stream is one LZ4BlockOutputStream whose content arrives in pieces: whatever the pieces and the room, its concatenated
output must be b200lz4block_compress_dev's stream of the whole content (no FLUSH, pieces at the whole content's phase), or
the stream LZ4BlockOutputStream writes with syncFlush (assembled here from the library's block compressor).  Each reader
stream is one LZ4BlockInputStream whose bytes arrive in pieces: its concatenated content, final status and total consumed
must be what b200lz4block_decompress_host gives for the whole stream, and on an error the content delivered in front of it
what a block-by-block restatement of refill() delivers.  Runs on the H100, and on the CPU emulator build of the library
(B200LZ4_TEST_SO=.../libb200lz4_sim*.so), where the sizes shrink and torch is not used."""
import ctypes
import os
import random

import numpy as np
import pytest

from test_frame_reader_dev import _cuts as _read_cuts, _rooms as _read_rooms
from test_frame_writer_dev import _cuts as _write_cuts, _place
from test_lz4block_dev import (_DevMem, _aligned, _check_layout, _faulty_streams, _header, _host_read, _lay_out, _level, _u64,
                               _write, SEED)

pytestmark = pytest.mark.gpu

SIM = "sim" in os.environ.get("B200LZ4_TEST_SO", "")
E_ARG = -2147483645
GUARD = 0xAA
MORE_INPUT, MORE_ROOM, DONE = 0, 1, 2
WRITE, FLUSH, CLOSE = 0, 1, 2
H = 21


class _Writer:
    def __init__(self, L, ns, bs, hc=0):
        self.L, err = L, ctypes.c_int(0)
        self.h = L.b200lz4block_writer_create(ns, bs, hc, ctypes.byref(err))
        assert self.h and err.value == 0, err.value

    def write(self, M, d_src, offs, lens, ops, d_dst, doff, dcap, stream=None):
        ns = len(lens)
        st = np.zeros(ns, dtype=np.int32)
        used, prod, need = (np.zeros(ns, dtype=np.uint64) for _ in range(3))
        o = np.ascontiguousarray(np.asarray(ops, dtype=np.uint8))
        rc = self.L.b200lz4block_writer_write_dev(self.h, M.ptr(d_src), offs.ctypes.data, lens.ctypes.data, o.ctypes.data,
                                                  M.ptr(d_dst), doff.ctypes.data, dcap.ctypes.data, st.ctypes.data,
                                                  used.ctypes.data, prod.ctypes.data, need.ctypes.data, stream)
        return rc, st, used, prod, need

    def free(self):
        self.L.b200lz4block_writer_free(self.h)


class _Reader:
    def __init__(self, L, ns, stop):
        self.L, err = L, ctypes.c_int(0)
        self.h = L.b200lz4block_reader_create(ns, int(stop), ctypes.byref(err))
        assert self.h and err.value == 0, err.value

    def read(self, M, d_src, offs, lens, eof, d_dst, doff, dcap, stream=None):
        ns = len(lens)
        st = np.zeros(ns, dtype=np.int32)
        used, prod, need = (np.zeros(ns, dtype=np.uint64) for _ in range(3))
        e = np.ascontiguousarray(np.asarray(eof, dtype=np.uint8))
        rc = self.L.b200lz4block_reader_read_dev(self.h, M.ptr(d_src), offs.ctypes.data, lens.ctypes.data, e.ctypes.data,
                                                 M.ptr(d_dst), doff.ctypes.data, dcap.ctypes.data, st.ctypes.data,
                                                 used.ctypes.data, prod.ctypes.data, need.ctypes.data, stream)
        return rc, st, used, prod, need

    def free(self):
        self.L.b200lz4block_reader_free(self.h)


def _ranges(caps):
    """destination ranges with 24 guard bytes in front of, between and behind them"""
    doff, q = [], 24
    for c in caps:
        doff.append(q)
        q += c + 24
    return doff, q + 64


def _drive_writer(L, M, datas, bs, cut, room, op=None, hc=0, phase=0, max_calls=200000, on_call=None):
    """every stream in one writer, one call per round until all are DONE (and one round more): stream k's piece is cut(k,
    rest, status, need, left) bytes from where it stopped, placed at phase + position (mod 16), with room(k, status, need,
    room); op(k, covers_rest, status) (default: CLOSE once the piece covers the rest).  On every call the guards hold,
    produced <= room, need > 0 on MORE_*, a DONE stream takes and produces nothing.  -> (outputs, flush points, calls)"""
    ns = len(datas)
    wr = _Writer(L, ns, bs, hc)
    pos, left, rooms = [0] * ns, [0] * ns, [0] * ns
    outs = [bytearray() for _ in datas]
    status, need, flushes = [None] * ns, [0] * ns, [[] for _ in datas]
    calls, after = 0, 0
    op = op or (lambda k, covers, s: CLOSE if covers else WRITE)
    while True:
        if all(s == DONE for s in status):
            if after:
                break
            after = 1
        pieces, ops, caps = [], [], []
        for k, d in enumerate(datas):
            rest = len(d) - pos[k]
            p = min(rest, max(cut(k, rest, status[k], need[k], left[k]), 0))
            rooms[k] = max(room(k, status[k], need[k], rooms[k]), 0)
            pieces.append(d[pos[k]:pos[k] + p])
            ops.append(op(k, p == rest, status[k]))
            caps.append(rooms[k])
        src, offs, lens = _place(pieces, [(phase + p) % 16 for p in pos])
        doff, total = _ranges(caps)
        d_dst = M.full(total, GUARD)
        rc, st, used, prod, nd = wr.write(M, M.up(src), offs, lens, ops, d_dst, _u64(doff), _u64(caps))
        assert rc == 0, rc
        calls += 1
        dst = M.down(d_dst)
        assert (dst[:24] == GUARD).all()
        for k in range(ns):
            s, u, pr, o = int(st[k]), int(used[k]), int(prod[k]), doff[k]
            if status[k] == DONE:
                assert s == DONE and u == 0 and pr == 0, (k, s, u, pr)
            assert u <= len(pieces[k]) and pr <= caps[k], (k, u, len(pieces[k]), pr, caps[k])
            assert (dst[o + pr:o + caps[k] + 24] == GUARD).all(), (k, s, pr, caps[k])
            outs[k] += dst[o:o + pr].tobytes()
            pos[k] += u
            left[k] = len(pieces[k]) - u
            if s in (MORE_INPUT, MORE_ROOM):
                assert int(nd[k]) > 0, (k, s)
            if ops[k] == FLUSH and s == MORE_INPUT:
                flushes[k].append(pos[k])
            status[k], need[k] = s, int(nd[k])
        if on_call is not None:
            on_call(st, used, prod, dst, doff)
        assert calls <= max_calls, (calls, status)
    wr.free()
    assert all(p == len(d) for p, d in zip(pos, datas))
    return outs, flushes, calls


def _expected(b200, port, data, flushes, bs, phase=0):
    """LZ4BlockOutputStream's stream for `data` with syncFlush and flush() at each offset of `flushes`
    (LZ4BlockOutputStream.java:160-266): blocks of bs between flushes, a short one at each flush, each compressed by this
    library's fast block compressor at its phase, as the writer runs it"""
    lvl, out = _level(bs), bytearray()
    cuts, a = [], 0
    for e in sorted(set(flushes)) + [len(data)]:
        cuts += [(o, min(bs, e - o)) for o in range(a, e, bs)]
        a = max(a, e)
    if cuts:
        offs = np.asarray([o for o, _ in cuts], dtype=np.uint64)
        lens = np.asarray([n for _, n in cuts], dtype=np.int32)
        cap = lens + lens // 255 + 16
        slot = (cap.astype(np.uint64) + 15) // 16 * 16
        coff = np.cumsum(slot) - slot
        comp = np.zeros(int(slot.sum()), dtype=np.uint8)
        clen = b200.batch.compress_fast_batch_host(_aligned(data, phase), offs, lens, comp, coff, cap,
                                                   max_src_len=65536 if bs <= 65536 else 0)
        for (o, n), co, c in zip(cuts, coff.tolist(), clen.tolist()):
            block = data[o:o + n]
            stored = c <= 0 or c >= n
            payload = block if stored else comp[co:co + c].tobytes()
            out += _header(0x10 if stored else 0x20, lvl, len(payload), n, port.xxh32(block, SEED) & 0x0FFFFFFF) + payload
    return bytes(out + _header(0x10, lvl, 0, 0, 0))


def _compress_dev(L, M, datas, bs, hc=0, phase=0):
    src, offs, lens = _place(datas, [phase] * len(datas))
    rc, d_dst, so, sl = _write(L, M, M.up(src), offs, lens, bs, hc)
    assert rc >= 0, rc
    out = M.down(d_dst)
    return [out[int(o):int(o) + int(n)].tobytes() for o, n in zip(so, sl)]


def _write_rooms(ample, rng):
    return {
        "ample": lambda k, s, need, r: ample[k],
        "exact": lambda k, s, need, r: need if s == MORE_ROOM else r,
        "tight": lambda k, s, need, r: need + rng.randrange(0, 2 * H) if s == MORE_ROOM else rng.randrange(0, 2 * H),
    }


def _datas(port):
    base = port.datagen(300000, 0.5, 0.0, 11).tobytes()
    rng = random.Random(4)
    lens = (0, 1, 63, 64, 65, 1000, 3000, 70000) if SIM else (0, 1, 63, 64, 65, 1000, 65535, 65536, 65537, 200000, 300000)
    return [base[:n] if k % 3 else rng.randbytes(n) for k, n in enumerate(lens)]


def _block_sizes():
    return (64, 1000, 65536, 65537) if SIM else (64, 1000, 4096, 65536, 65537, 1 << 20)


@pytest.mark.parametrize("phase", [0, 5])
def test_writer_whole_content_parity(b200, port, phase):
    """block sizes 64, 1000 (not a power of two), 65 536 and one above 64 KiB, cut at random, at need and at need -1 / +1 and
    whole, with ample, exact and tight room spread over the streams, each piece at the whole content's phase plus what was
    taken: every stream's output is b200lz4block_compress_dev's stream of the whole content; short streams dripped one
    byte at a time too"""
    L, M = b200._native.lib(), _DevMem()
    datas = _datas(port)
    rng = random.Random(3 + phase)
    cuts = _write_cuts(rng)
    names = ["random", "need", "need-1+1", "whole"]
    for bi, bs in enumerate(_block_sizes()):
        ds = [d for d in datas if len(d) <= 20 * bs] if SIM else datas
        want = _compress_dev(L, M, ds, bs, phase=phase)
        ample = [L.b200lz4block_compress_bound(len(d), bs) for d in ds]
        rooms = _write_rooms(ample, rng)
        for cn in ((names[(bi + phase) % 4],) if SIM else names):
            rn = [("ample", "exact", "tight")[(k + bi) % 3] for k in range(len(ds))]
            outs, _, _ = _drive_writer(L, M, ds, bs, cuts[cn], lambda k, *a: rooms[rn[k]](k, *a), phase=phase)
            for k, (o, w) in enumerate(zip(outs, want)):
                assert bytes(o) == w, (bs, cn, k, len(ds[k]))
    short = [d for d in datas if len(d) <= 70]
    for bs in (64, 65536):
        want = _compress_dev(L, M, short, bs, phase=phase)
        outs, _, _ = _drive_writer(L, M, short, bs, cuts["drip"], lambda k, s, need, r: need if s == MORE_ROOM else r, phase=phase)
        assert [bytes(o) for o in outs] == want, bs


def test_writer_flush_parity_and_read_back(b200, port):
    """FLUSH at random points, FLUSH with nothing left and CLOSE right after a FLUSH: the output is the stream
    LZ4BlockOutputStream writes with syncFlush, and it reads back to the content with both stopOnEmptyBlock values, through
    the host reader and the incremental reader"""
    L, M = b200._native.lib(), _DevMem()
    rng = random.Random(7)
    datas = _datas(port)
    for bs in ((1000, 65536) if SIM else (1000, 65536, 65537)):
        ample = [L.b200lz4block_compress_bound(len(d), bs) + H * (len(d) // 500 + 8) for d in datas]

        def op(k, covers, s):
            r = rng.random()
            return (CLOSE if r < 0.5 else FLUSH) if covers else (FLUSH if r < 0.35 else WRITE)

        def cut(k, rest, s, need, left):
            return left + rng.choice([0, 1, 17, 1000, 70000, need or 1, rest])

        outs, flushes, _ = _drive_writer(L, M, datas, bs, cut, lambda k, s, need, r: ample[k] if k % 2 else (need if s == MORE_ROOM else r),
                                         op=op, phase=3)
        assert any(flushes)
        blobs = [bytes(o) for o in outs]
        for k, (o, d) in enumerate(zip(blobs, datas)):
            assert o == _expected(b200, port, d, flushes[k], bs, phase=3), (bs, k, flushes[k])
            for stop in (True, False):
                assert _host_read(L, o, len(d), stop)[::2] == (len(d), d), (bs, k, stop)
        for stop in (True, False):
            status, got, _, _ = _drive_reader(L, M, blobs, stop, lambda k, rest, s, need, p: rest,
                                              lambda k, s, need, r: max(len(d) for d in datas) + 1)
            assert status == [DONE] * len(datas) and [bytes(g) for g in got] == datas, (bs, stop)


def test_writer_high_compressor(b200, port):
    """hc_level 9, cut at random, room exact: the streams have the layout and checksums LZ4BlockOutputStream writes and read
    back; on the emulator, where HC's order is fixed, they are b200lz4block_compress_dev's at the same level"""
    L, M = b200._native.lib(), _DevMem()
    datas = [port.datagen(n, 0.5, 0.0, 5 + n % 7).tobytes() for n in ((5000, 1, 0) if SIM else (300000, 65537, 1, 0))]
    bs = 1000 if SIM else 65536
    want = _compress_dev(L, M, datas, bs, hc=9)
    outs, _, _ = _drive_writer(L, M, datas, bs, _write_cuts(random.Random(2))["random"],
                               lambda k, s, need, r: need if s == MORE_ROOM else r, hc=9)
    for o, w, d in zip(outs, want, datas):
        _check_layout(port, bytes(o), d, bs)
        assert port.lz4block_decompress(bytes(o), len(d)) == (len(d), d)
        if SIM:
            assert bytes(o) == w


def test_writer_edge_cases(b200, port):
    """CLOSE on an empty stream writes exactly one end block; FLUSH with nothing left writes nothing; MORE_ROOM's need is
    21 + the block's length (21 for the end block) and a call given exactly that progresses; MORE_INPUT's need is what the
    next whole block lacks, blockSize after a flush; DONE is latched"""
    L, M = b200._native.lib(), _DevMem()
    data = port.datagen(5000, 0.5, 0.0, 3).tobytes()
    bs = 1000

    def step(wr, piece, op, cap, at=0):
        src, offs, lens = _place([piece], [at % 16])
        d_dst = M.full(cap + 64, GUARD)
        rc, st, used, prod, need = wr.write(M, M.up(src), offs, lens, [op], d_dst, _u64([0]), _u64([cap]))
        out = M.down(d_dst)
        assert rc == 0 and (out[int(prod[0]):] == GUARD).all()
        return int(st[0]), int(used[0]), int(prod[0]), int(need[0]), out[:int(prod[0])].tobytes()

    for bsz in (64, 1 << 20):
        wr = _Writer(L, 1, bsz)
        st, used, prod, need, out = step(wr, b"", CLOSE, H - 1)
        assert (st, used, prod, need) == (MORE_ROOM, 0, 0, H)
        st, used, prod, need, out = step(wr, b"", CLOSE, 100)
        assert (st, used, need) == (DONE, 0, 0) and out == _header(0x10, _level(bsz), 0, 0, 0) == _compress_dev(L, M, [b""], bsz)[0]
        assert step(wr, data[:100], CLOSE, 1000) == (DONE, 0, 0, 0, b"")
        assert step(wr, data[:100], WRITE, 1000) == (DONE, 0, 0, 0, b"")
        wr.free()
    wr = _Writer(L, 1, bs)
    got = bytearray()
    assert step(wr, data[:10], WRITE, 0)[:4] == (MORE_INPUT, 0, 0, bs - 10)
    assert step(wr, b"", FLUSH, 50)[:4] == (MORE_INPUT, 0, 0, bs)                 # nothing left: nothing written
    assert step(wr, data[:bs + 5], WRITE, bs + H - 1)[:4] == (MORE_ROOM, 0, 0, bs + H)
    s = step(wr, data[:bs + 5], WRITE, bs + H)
    assert s[:2] == (MORE_INPUT, bs) and s[3] == bs - 5
    got += s[4]
    assert step(wr, data[bs:bs + 5], FLUSH, 5 + H - 1)[:4] == (MORE_ROOM, 0, 0, 5 + H)
    s = step(wr, data[bs:bs + 5], FLUSH, 5 + H)
    assert s[:2] == (MORE_INPUT, 5) and s[3] == bs
    got += s[4]
    assert step(wr, b"", FLUSH, 0)[:4] == (MORE_INPUT, 0, 0, bs)
    s = step(wr, data[bs + 5:bs + 64], CLOSE, 59 + 2 * H - 1, at=bs + 5)        # the block fits, the end block does not
    assert s[:2] == (MORE_ROOM, 59) and s[3] == H and s[2] <= 59 + H
    got += s[4]
    s = step(wr, b"", CLOSE, H)
    assert s[:4] == (DONE, 0, H, 0)
    got += s[4]
    assert bytes(got) == _expected(b200, port, data[:bs + 64], [bs + 5], bs)
    wr.free()


# ---- reader
def _refill(port, blob, stop):
    """LZ4BlockInputStream.refill block by block (LZ4BlockInputStream.java:191-264; each block through the oracle's reader
    on its own) -> (code or total, the content delivered before it stopped, the summed original lengths of the blocks whose
    header it read: room enough for the whole stream)"""
    out, ip, n, room = bytearray(), 0, len(blob), 0
    while True:
        if n - ip < H:
            return (-1 if stop else len(out)), bytes(out), room
        h = blob[ip:ip + H]
        token = h[8]
        method, level = token & 0xF0, 10 + (token & 0x0F)
        clen, olen = int.from_bytes(h[9:13], "little", signed=True), int.from_bytes(h[13:17], "little", signed=True)
        check = int.from_bytes(h[17:21], "little")
        if h[:8] != b"LZ4Block" or method not in (0x10, 0x20) or olen > 1 << level or olen < 0 or clen < 0 or \
                (olen == 0) != (clen == 0) or (method == 0x10 and olen != clen):
            return -2, bytes(out), room
        ip += H
        if olen == 0:
            if check != 0:
                return -2, bytes(out), room
            if stop:
                return len(out), bytes(out), room
            continue
        room += olen
        if n - ip < clen:
            return -1, bytes(out), room
        r, dec = port.lz4block_decompress(h + blob[ip:ip + clen] + _header(0x10, token & 0x0F, 0, 0, 0), olen, True)
        if r != olen:
            return -2, bytes(out), room
        out += dec
        ip += clen


def _drive_reader(L, M, blobs, stop, cut, room, max_calls=100000, extra=1):
    """every stream in one reader, one call per round: stream k's piece is cut(k, rest, status, need, piece) bytes from where
    it stopped, its room room(k, status, need, room).  Each call's guard bytes around every range, and behind the produced
    part of a stream without an error, must be untouched, and a latched stream takes and produces nothing.  -> (status,
    content, consumed, calls)"""
    ns = len(blobs)
    rd = _Reader(L, ns, stop)
    pos, piece, rooms = [0] * ns, [0] * ns, [0] * ns
    outs = [bytearray() for _ in blobs]
    status, need = [None] * ns, [0] * ns
    calls, after = 0, 0
    while True:
        if all(s is not None and (s < 0 or s == DONE) for s in status):
            if after == extra:
                break
            after += 1
        pieces, eof, caps = [], [], []
        for k, b in enumerate(blobs):
            rest = len(b) - pos[k]
            p = min(rest, max(cut(k, rest, status[k], need[k], piece[k]), 0))
            rooms[k] = max(room(k, status[k], need[k], rooms[k]), 0)
            piece[k] = p
            pieces.append(b[pos[k]:pos[k] + p])
            eof.append(p == rest)
            caps.append(rooms[k])
        src, offs, lens = _lay_out(pieces, align=16, phase=5, gap=3)
        doff, total = _ranges(caps)
        d_dst = M.full(total, GUARD)
        rc, st, used, prod, nd = rd.read(M, M.up(src), offs, lens, eof, d_dst, _u64(doff), _u64(caps))
        assert rc == 0, rc
        calls += 1
        dst = M.down(d_dst)
        assert (dst[:24] == GUARD).all()
        for k in range(ns):
            s, u, pr, o = int(st[k]), int(used[k]), int(prod[k]), doff[k]
            if status[k] is not None and (status[k] < 0 or status[k] == DONE):
                assert s == status[k] and u == 0 and pr == 0, (k, s, status[k], u, pr)
            assert u <= piece[k] and pr <= caps[k], (k, u, piece[k], pr, caps[k])
            assert (dst[o + (caps[k] if s < 0 else pr):o + caps[k] + 24] == GUARD).all(), (k, s, pr, caps[k])
            outs[k] += dst[o:o + pr].tobytes()
            pos[k] += u
            status[k], need[k] = s, int(nd[k])
            if s in (MORE_INPUT, MORE_ROOM):
                assert need[k] > 0, (k, s)
            else:
                assert need[k] == 0, (k, s)
        assert calls <= max_calls, (calls, status)
    rd.free()
    return status, outs, pos, calls


def _check(L, port, blobs, stop, status, outs, pos, seen=None):
    for k, b in enumerate(blobs):
        want, h_used, h_out = _host_read(L, b, 1 << 24, stop)
        code, delivered, _ = _refill(port, b, stop)
        assert code == want, (k, code, want)
        if want >= 0:
            assert status[k] == DONE and outs[k] == h_out and pos[k] == h_used, (stop, k, status[k], len(outs[k]), want, pos[k], h_used)
        else:
            assert status[k] == want and outs[k] == delivered, (stop, k, status[k], want, len(outs[k]), len(delivered))
        if seen is not None:
            seen[want if want < 0 else "ok"] = seen.get(want if want < 0 else "ok", 0) + 1


def _parity(b200, port, stop, cut_names, room_names, short_only=False):
    L, M = b200._native.lib(), _DevMem()
    blobs = [b for b, _ in _faulty_streams(port, random.Random(77 + stop), 12 if SIM else 300)]
    if short_only:
        blobs = [b for b in blobs if len(b) <= (300 if SIM else 20000)]
    ample = [max(_refill(port, b, stop)[2], 1) for b in blobs]
    cuts, rooms = _read_cuts(random.Random(5)), _read_rooms(ample)
    seen = {}
    for ci, cn in enumerate(cut_names):
        rn = [room_names[(k + ci) % len(room_names)] for k in range(len(blobs))]
        status, outs, pos, _ = _drive_reader(L, M, blobs, stop, lambda k, *a: cuts[cn](k, *a), lambda k, *a: rooms[rn[k]](k, *a),
                                             extra=2)
        _check(L, port, blobs, stop, status, outs, pos, seen)
    return seen


@pytest.mark.parametrize("stop", [True, False])
def test_reader_split_parity_on_faulty_streams(b200, port, stop):
    """the faulty streams of test_lz4block_dev (truncated, bit-flipped, concatenated, without end blocks, empty, garbage) read
    whole, cut at random past each unit, at exactly need and at need -1 / +1 (the emulator: the last only), with ample, exact
    and growing-from-zero room spread over the streams: status, content and total consumed are the host reader's; on an
    error the content delivered is the restated refill()'s; guards hold on every call and latched streams stay put"""
    cuts = ["need-1+1"] if SIM else ["whole", "random", "need", "need-1+1"]
    seen = _parity(b200, port, stop, cuts, ["ample", "exact", "growing"])
    assert {"ok", -1, -2} <= set(seen), seen


@pytest.mark.parametrize("stop", [True, False])
def test_reader_split_parity_one_byte_drip(b200, port, stop):
    """the short streams of the same corpus fed one byte more per call"""
    _parity(b200, port, stop, ["drip"], ["exact", "growing"], short_only=True)


def test_reader_concatenated_writer_streams(b200, port):
    """streams of the incremental writer, flushed at random, laid back to back and read as one stream with stopOnEmptyBlock
    false, cut at random: the contents come back concatenated; with it true the first stream comes back"""
    L, M = b200._native.lib(), _DevMem()
    rng = random.Random(9)
    datas = [d for d in _datas(port) if len(d) <= 70000]
    outs, _, _ = _drive_writer(L, M, datas, 1000, lambda k, rest, s, need, left: left + rng.randrange(0, 3000),
                               lambda k, s, need, r: 1 << 17, op=lambda k, covers, s: CLOSE if covers else rng.choice([WRITE, FLUSH]))
    blob = b"".join(bytes(o) for o in outs)
    cuts = _read_cuts(random.Random(3))
    for stop, want in ((False, b"".join(datas)), (True, datas[0])):
        status, got, pos, _ = _drive_reader(L, M, [blob], stop, cuts["random"], lambda k, s, need, r: 1 << 17)
        assert status == [DONE] and bytes(got[0]) == want, stop
        assert pos[0] == (len(blob) if not stop else len(outs[0]))


def test_reader_edge_cases(b200, port):
    """need on MORE_INPUT is 21 until a header is readable, then 21 + its compressed length; need on MORE_ROOM is the block's
    original length and a call given exactly that progresses; with room for the largest block and the whole rest presented,
    a stream finishes in at most its block count + 2 calls; DONE and errors are latched"""
    L, M = b200._native.lib(), _DevMem()
    data = port.datagen(5000, 0.5, 0.0, 8).tobytes()
    blob = b200.compress_lz4block(data, 1000)
    units, ip = [], 0
    while ip < len(blob):
        clen, olen = int.from_bytes(blob[ip + 9:ip + 13], "little"), int.from_bytes(blob[ip + 13:ip + 17], "little")
        units.append((ip, clen, olen))
        ip += H + clen
    rd = _Reader(L, 1, True)

    def step(piece, cap, eof=False):
        src = np.frombuffer(piece + bytes(16), dtype=np.uint8)
        d_dst = M.full(cap + 64, GUARD)
        rc, st, used, prod, need = rd.read(M, M.up(src), _u64([0]), _u64([len(piece)]), [eof], d_dst, _u64([0]), _u64([cap]))
        out = M.down(d_dst)
        assert rc == 0 and (out[cap if int(st[0]) < 0 else int(prod[0]):] == GUARD).all()
        return int(st[0]), int(used[0]), int(prod[0]), int(need[0]), out[:int(prod[0])].tobytes()

    (a0, c0, o0), (a1, c1, o1) = units[0], units[1]
    assert step(blob[:H - 1], 5000)[:4] == (MORE_INPUT, 0, 0, H)
    assert step(blob[:H + c0 - 1], 5000)[:4] == (MORE_INPUT, 0, 0, H + c0)
    assert step(blob[:H + c0], o0 - 1)[:4] == (MORE_ROOM, 0, 0, o0)
    s = step(blob[:H + c0 + 3], o0)
    assert s[:4] == (MORE_INPUT, H + c0, o0, H) and s[4] == data[:o0]
    rd.free()
    for stop in (True, False):
        status, outs, pos, calls = _drive_reader(L, M, [blob], stop, lambda k, rest, s, need, p: rest,
                                                 lambda k, s, need, r: 1000, extra=0)
        assert status == [DONE] and bytes(outs[0]) == data and pos[0] == len(blob) and calls <= len(units) + 2, (stop, calls)
    # latching: an error, then DONE
    bad = bytearray(blob)
    bad[a1 + H] ^= 0xFF
    for b, want in ((bytes(bad), -2), (blob, DONE)):
        rd = _Reader(L, 1, True)
        s = step(b, 5000, True)
        assert s[0] == want and s[2] == (o0 if want < 0 else len(data)) and s[1] == (a1 if want < 0 else len(blob)), s[:4]
        assert step(b, 5000, True)[:4] == (want, 0, 0, 0)
        assert step(b"", 0, False)[:4] == (want, 0, 0, 0)
        rd.free()


def test_errors_launch_nothing_and_write_nothing(b200, port):
    """create: blockSize 63 and 32 MiB + 1, ns above 2^31 - 1 give NULL and B200LZ4_E_ARG.  write / read: a NULL handle or
    pointer, an op above CLOSE, a destination range that overflows give B200LZ4_E_ARG before anything is launched or
    written, and the streams' states are unchanged; handles of 0 streams return 0"""
    L, M = b200._native.lib(), _DevMem()
    err = ctypes.c_int(0)
    for args in ((1, 63, 0), (1, (1 << 25) + 1, 0), (1 << 31, 65536, 0)):
        assert not L.b200lz4block_writer_create(*args, ctypes.byref(err)) and err.value == E_ARG, args
    assert not L.b200lz4block_reader_create(1 << 31, 1, ctypes.byref(err)) and err.value == E_ARG
    data = port.datagen(100000, 0.5, 0.0, 6).tobytes()
    src, offs, lens = _place([data, b"xyz"], [0, 0])
    d_src, d_dst = M.up(src), M.full(300100, GUARD)
    doff, dcap = _u64([0, 200000]), _u64([150000, 100])
    z = np.zeros(2, dtype=np.uint64)
    st = np.zeros(2, dtype=np.int32)
    last = np.full(2, CLOSE, dtype=np.uint8)
    wr, rd = _Writer(L, 2, 65536), _Reader(L, 2, True)
    before = L.b200lz4_launch_count()
    args = [M.ptr(d_src), offs.ctypes.data, lens.ctypes.data, last.ctypes.data, M.ptr(d_dst), doff.ctypes.data, dcap.ctypes.data,
            st.ctypes.data, z.ctypes.data, z.ctypes.data, z.ctypes.data, None]
    for fn, h in ((L.b200lz4block_writer_write_dev, wr.h), (L.b200lz4block_reader_read_dev, rd.h)):
        assert fn(None, *args) == E_ARG
        for i in range(11):
            bad = list(args)
            bad[i] = None
            assert fn(h, *bad) == E_ARG, i
        bad = list(args)
        far = _u64([0, (1 << 64) - 50])
        bad[5] = far.ctypes.data
        assert fn(h, *bad) == E_ARG
    bad = list(args)
    bad[3] = np.asarray([CLOSE, 3], dtype=np.uint8).ctypes.data
    assert L.b200lz4block_writer_write_dev(wr.h, *bad) == E_ARG
    assert L.b200lz4_launch_count() == before and (M.down(d_dst) == GUARD).all()
    for create, fn, free in ((lambda: L.b200lz4block_writer_create(0, 65536, 0, ctypes.byref(err)), L.b200lz4block_writer_write_dev,
                              L.b200lz4block_writer_free),
                             (lambda: L.b200lz4block_reader_create(0, 1, ctypes.byref(err)), L.b200lz4block_reader_read_dev,
                              L.b200lz4block_reader_free)):
        empty = create()
        assert empty and fn(empty, *([None] * 12)) == 0
        free(empty)
    rc, s, used, prod, need = wr.write(M, d_src, offs, lens, [CLOSE, CLOSE], d_dst, doff, dcap)
    assert rc == 0 and s.tolist() == [DONE, DONE] and used.tolist() == [len(data), 3]
    out = M.down(d_dst)
    streams = [out[:int(prod[0])].tobytes(), out[200000:200000 + int(prod[1])].tobytes()]
    assert streams == _compress_dev(L, M, [data, b"xyz"], 65536)
    s2, o2, l2 = _place(streams, [0, 0])
    d_out = M.full(200064, GUARD)
    rc, s, used, prod, need = rd.read(M, M.up(s2), o2, l2, [True, True], d_out, _u64([0, 150000]), _u64([100000, 100]))
    assert rc == 0 and s.tolist() == [DONE, DONE] and prod.tolist() == [len(data), 3] and used.tolist() == [len(b) for b in streams]
    wr.free()
    rd.free()


def test_launches_do_not_depend_on_streams_or_blocks(b200, port):
    """the writer: one stream of n blocks and n streams of one block; the reader: the same n blocks as one stream and as n
    streams, and one stream of 2n blocks: each launches the same kernels"""
    L, M = b200._native.lib(), _DevMem()
    n, bs = (8, 4096) if SIM else (64, 65536)
    body = port.datagen(2 * n * bs, 0.5, 0.0, 7).tobytes()
    wcounts, streams = [], []
    for datas in ([body[:n * bs]], [body[k * bs:(k + 1) * bs] for k in range(n)]):
        src, offs, lens = _place(datas, [0] * len(datas))
        wr = _Writer(L, len(datas), bs)
        caps = [L.b200lz4block_compress_bound(len(d), bs) for d in datas]
        doff, total = _ranges(caps)
        d_dst = M.full(total, 0)
        b = L.b200lz4_launch_count()
        rc, s, used, prod, need = wr.write(M, M.up(src), offs, lens, [CLOSE] * len(datas), d_dst, _u64(doff), _u64(caps))
        wcounts.append(L.b200lz4_launch_count() - b)
        assert rc == 0 and (s == DONE).all()
        out = M.down(d_dst)
        streams.append([out[o:o + int(p)].tobytes() for o, p in zip(doff, prod)])
        wr.free()
    assert wcounts[0] == wcounts[1], wcounts
    rcounts = []
    for blobs in (streams[0], streams[1], _compress_dev(L, M, [body], bs)):
        src, offs, lens = _place(blobs, [0] * len(blobs))
        rd = _Reader(L, len(blobs), True)
        caps = [len(body)] * len(blobs)
        doff, total = _ranges(caps)
        d_dst = M.full(total, 0)
        b = L.b200lz4_launch_count()
        rc, s, used, prod, need = rd.read(M, M.up(src), offs, lens, [True] * len(blobs), d_dst, _u64(doff), _u64(caps))
        rcounts.append(L.b200lz4_launch_count() - b)
        assert rc == 0 and (s == DONE).all()
        rd.free()
    assert rcounts[0] == rcounts[1] == rcounts[2], rcounts


def _counted(L):
    if not hasattr(L, "b200lz4_sim_device_bytes"):
        pytest.skip("this emulator library does not count copies and allocations: tests/simt/alloc_count.h")
    L.b200lz4_sim_copied_bytes.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
    L.b200lz4_sim_device_bytes.argtypes = [ctypes.c_void_p, ctypes.c_void_p]


@pytest.mark.skipif(not SIM, reason="the counting emulator build counts the library's host<->device copies")
def test_per_call_copies_do_not_depend_on_payload(b200, port):
    """the same streams and block counts at block sizes 1 KiB and 16 KiB, written with WRITE, FLUSH and CLOSE and read back
    in the same pieces: every call copies the same bytes between host and device"""
    L, M = b200._native.lib(), _DevMem()
    _counted(L)
    h2d, d2h = ctypes.c_ulonglong(0), ctypes.c_ulonglong(0)

    def copied(fn):
        L.b200lz4_sim_copied_bytes(ctypes.byref(h2d), ctypes.byref(d2h))
        a = (h2d.value, d2h.value)
        r = fn()
        L.b200lz4_sim_copied_bytes(ctypes.byref(h2d), ctypes.byref(d2h))
        return r, (h2d.value - a[0], d2h.value - a[1])

    counts = {"write": [], "read": []}
    for bs in (1024, 16384):
        rng = random.Random(8)
        datas = [rng.randbytes(3 * bs + 100) for _ in range(3)]
        wr, rd = _Writer(L, len(datas), bs), _Reader(L, len(datas), True)
        pos = [0] * len(datas)
        for rnd, op in enumerate((WRITE, FLUSH, CLOSE)):
            pieces = [d[p:p + (bs if rnd == 0 else 2 * bs + (100 if op == CLOSE else 0))] for d, p in zip(datas, pos)]
            src, offs, lens = _place(pieces, [0] * len(pieces))
            caps = [4 * bs] * len(datas)
            doff, total = _ranges(caps)
            d_dst = M.full(total, 0)
            (rc, st, u, prod, need), c = copied(lambda: wr.write(M, M.up(src), offs, lens, [op] * len(datas), d_dst, _u64(doff), _u64(caps)))
            counts["write"].append((rnd, c))
            assert rc == 0
            pos = [p + int(x) for p, x in zip(pos, u)]
            out = M.down(d_dst)
            blobs = [out[o:o + int(p)].tobytes() for o, p in zip(doff, prod)]
            s2, o2, l2 = _place(blobs, [0] * len(blobs))
            d_out = M.full(total, 0)
            (rc, st, u, prod, need), c = copied(lambda: rd.read(M, M.up(s2), o2, l2, [op == CLOSE] * len(datas), d_out, _u64(doff), _u64(caps)))
            counts["read"].append((rnd, c))
            assert rc == 0 and (u == l2).all()
        wr.free()
        rd.free()
    for fn, c in counts.items():
        assert c[:3] == c[3:], (fn, c)
        assert max(sum(x[1]) for x in c) < 4096, (fn, c)


@pytest.mark.skipif(not SIM, reason="the counting emulator build counts the library's device allocations")
def test_device_memory_does_not_grow_with_the_stream(b200, port):
    """one stream written 4 blocks per call and each call's output read at once by a reader: 16 blocks take less than 1 MiB
    of device scratch, and 64 blocks written and read behind them allocate nothing more"""
    L, M = b200._native.lib(), _DevMem()
    _counted(L)
    bs = 4096
    content = port.datagen(bs, 0.5, 0.0, 4).tobytes()
    grown = []
    for nblocks in (16, 64):
        live, peak = ctypes.c_ulonglong(0), ctypes.c_ulonglong(0)
        L.b200lz4_sim_reset_device_peak()
        L.b200lz4_sim_device_bytes(ctypes.byref(live), ctypes.byref(peak))
        base = live.value
        rd = _Reader(L, 1, True)
        got = bytearray()

        def on_call(st, used, prod, dst, doff):
            piece = dst[doff[0]:doff[0] + int(prod[0])].tobytes()
            src = np.frombuffer(piece + bytes(16), dtype=np.uint8)
            d_out = M.full(4 * bs, 0)
            rc, s, u, p, n = rd.read(M, M.up(src), _u64([0]), _u64([len(piece)]), [int(st[0]) == DONE], d_out, _u64([0]), _u64([4 * bs]))
            assert rc == 0 and int(u[0]) == len(piece)
            got.extend(M.down(d_out)[:int(p[0])].tobytes())

        _drive_writer(L, M, [content * nblocks], bs, lambda k, rest, s, need, left: left + 4 * bs, lambda k, s, need, r: 4 * (bs + H) + 64,
                      on_call=on_call)
        rd.free()
        L.b200lz4_sim_device_bytes(ctypes.byref(live), ctypes.byref(peak))
        grown.append(peak.value - base)
        assert bytes(got) == content * nblocks
    assert grown[0] < (1 << 20) and grown[1] == 0, grown


@pytest.mark.skipif(SIM, reason="device memory beyond the emulator's")
def test_stream_longer_than_the_card(b200, port):
    """one LZ4Block stream of 96 GiB of content at 64 KiB blocks: one 256 MiB device piece written again and again into one
    fixed output buffer, each call's output read at once by an incremental reader into one fixed content buffer, so the
    stream never exists anywhere whole; every piece read back has the source's XXH64, and the reader ends DONE"""
    import torch
    piece = torch.from_numpy(port.datagen(4 << 20, 0.5, 0.0, 17)).cuda().repeat(64)          # 256 MiB
    n = piece.numel()
    out = torch.empty(b200._native.lib().b200lz4block_compress_bound(n, 65536) + 64, dtype=torch.uint8, device="cuda")
    content = torch.empty(n, dtype=torch.uint8, device="cuda")

    def xxh64(buf, ln):
        h = torch.zeros(1, dtype=torch.int64, device="cuda")
        b200.batch.xxh64_batch_dev(buf, torch.zeros(1, dtype=torch.int64, device="cuda"),
                                   torch.tensor([ln], dtype=torch.int32, device="cuda"), h)
        return int(h.item())

    want = xxh64(piece, n)
    calls, produced = 96 * 4, 0
    with b200.LZ4BlockWriter(1, 1 << 16) as wr, b200.LZ4BlockReader(1) as rd:
        for c in range(calls + 1):
            close = c == calls
            st, used, prod, need = wr.write(piece, [0], [0 if close else n], out, [0], [out.numel()], [CLOSE if close else WRITE])
            assert int(st[0]) == (DONE if close else MORE_INPUT) and int(used[0]) == (0 if close else n), (c, st, used)
            p = int(prod[0])
            rs, ru, rp, _ = rd.read(out, [0], [p], content, [0], [n], [close])
            assert int(ru[0]) == p and int(rs[0]) == (DONE if close else MORE_INPUT), (c, rs, ru, p)
            if not close:
                assert int(rp[0]) == n and xxh64(content, n) == want, c
            produced += int(rp[0])
    assert produced == 96 << 30


@pytest.mark.skipif(SIM, reason="torch tensors and streams: GPU only")
def test_python_wrappers_and_stream_order(b200, port):
    """frame.LZ4BlockWriter / LZ4BlockReader against the C ABI, their argument checks, and sources written by torch ops on a
    side stream with both calls made on that stream without a synchronise: the streams hold the new bytes and read back"""
    import torch
    L, M = b200._native.lib(), _DevMem()
    old, new = port.datagen(3 << 20, 0.5, 0.0, 1), port.datagen(3 << 20, 0.5, 0.0, 2)
    d_src, d_new = M.up(old), M.up(new)
    out = torch.full((8 << 20,), GUARD, dtype=torch.uint8, device="cuda")
    back = torch.full((3 << 20,), GUARD, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    half = 3 << 19
    with b200.LZ4BlockWriter(2, 1 << 16) as wr, b200.LZ4BlockReader(2, stop_on_empty_block=True) as rd:
        with torch.cuda.stream(side):
            torch.cuda._sleep(20_000_000)                                   # the copy lands well after the calls are made
            d_src.copy_(d_new)
            st, used, prod, need = wr.write(d_src, [0, half], [half, half], out, [0, 4 << 20], [4 << 20, 4 << 20],
                                            [b200.frame.CLOSE, b200.frame.CLOSE])
            copy = torch.zeros_like(out)
            torch.cuda._sleep(20_000_000)
            copy.copy_(out)
            rs, ru, rp, rn = rd.read(copy, [0, 4 << 20], [int(prod[0]), int(prod[1])], back, [0, half], [half, half], [True, True])
        torch.cuda.synchronize()
        assert st.dtype == np.int32 and used.dtype == np.uint64 and prod.dtype == np.uint64 and need.dtype == np.uint64
        assert st.tolist() == [DONE, DONE] and used.tolist() == [half, half]
        host = out.cpu().numpy()
        got = [host[:int(prod[0])].tobytes(), host[4 << 20:(4 << 20) + int(prod[1])].tobytes()]
        assert got == _compress_dev(L, M, [new[:half].tobytes(), new[half:].tobytes()], 1 << 16)
        assert (host[int(prod[0]):4 << 20] == GUARD).all()
        assert rs.tolist() == [DONE, DONE] and ru.tolist() == prod.tolist() and rp.tolist() == [half, half]
        assert back.cpu().numpy().tobytes() == new.tobytes()
        with pytest.raises(ValueError):
            wr.write(d_src, [0], [1], out, [0], [1], [0])                      # one entry, two streams
        with pytest.raises(ValueError):
            wr.write(d_src.cpu(), [0, 0], [1, 1], out, [0, 0], [1, 1], [0, 0])
        with pytest.raises(ValueError):
            wr.write(d_src, [0, 0], [1, 1], out, [0, 0], [1, (8 << 20) + 1], [0, 0])
        with pytest.raises(ValueError):
            wr.write(d_src, [0, 0], [1, 1], out, [0, 0], [1, 1], [0, 3])
        with pytest.raises(ValueError):
            rd.read(d_src, [0, 0], [1, 1], out.cpu(), [0, 0], [1, 1], [True, True])
        with pytest.raises(ValueError):
            rd.read(d_src, [0, 0], [1, 1], out, [0, 0], [1, 1], [True])
    with pytest.raises(ValueError):
        wr.write(d_src, [0, 0], [1, 1], out, [0, 0], [1, 1], [0, 0])           # closed
    with pytest.raises(ValueError):
        rd.read(d_src, [0, 0], [1, 1], out, [0, 0], [1, 1], [True, True])
    with pytest.raises(ValueError):
        b200.LZ4BlockWriter(1, 63)
