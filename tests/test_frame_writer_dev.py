"""b200lz4f_writer_*: the incremental device frame writer.  Each stream is one LZ4FrameOutputStream whose content arrives in
pieces; a call writes the header on a stream's first call, takes whole blocks from the start of each piece, a short block at
FLUSH and the EndMark at CLOSE, and carries the stream's content checksum to the next call.  Whatever the pieces and the room,
the concatenated output must be the frame LZ4FrameOutputStream writes: without FLUSH and at the whole content's phase the one
b200lz4f_compress_dev writes, with FLUSH the one assembled here from the library's block compressor, and every reader must
read it back.  Runs on the H100, and on the CPU emulator build of the library (B200LZ4_TEST_SO=.../libb200lz4_sim*.so), where
the sizes shrink and torch is not used."""
import ctypes
import os
import random

import numpy as np
import pytest

from test_frame_encode_dev import _aligned, _mixed, _reference, _write
from test_frame_reader_dev import _Reader
from test_lz4block_dev import _DevMem, _u64

pytestmark = pytest.mark.gpu

SIM = "sim" in os.environ.get("B200LZ4_TEST_SO", "")
E_ARG = -2147483645
GUARD = 0xAA
MORE_INPUT, MORE_ROOM, DONE = 0, 1, 2
WRITE, FLUSH, CLOSE = 0, 1, 2


class _Writer:
    def __init__(self, L, ns, bs_code, flags, hc=0, known=None):
        self.L, err = L, ctypes.c_int(0)
        self.known = None if known is None else np.ascontiguousarray(np.asarray(known, dtype=np.int64))
        self.h = L.b200lz4f_writer_create(ns, bs_code, flags, hc, None if self.known is None else self.known.ctypes.data,
                                          ctypes.byref(err))
        assert self.h and err.value == 0, err.value

    def write(self, M, d_src, offs, lens, ops, d_dst, doff, dcap, stream=None):
        ns = len(lens)
        st = np.zeros(ns, dtype=np.int32)
        used, prod, need = (np.zeros(ns, dtype=np.uint64) for _ in range(3))
        o = np.ascontiguousarray(np.asarray(ops, dtype=np.uint8))
        rc = self.L.b200lz4f_writer_write_dev(self.h, M.ptr(d_src), offs.ctypes.data, lens.ctypes.data, o.ctypes.data, M.ptr(d_dst),
                                              doff.ctypes.data, dcap.ctypes.data, st.ctypes.data, used.ctypes.data,
                                              prod.ctypes.data, need.ctypes.data, stream)
        return rc, st, used, prod, need

    def free(self):
        self.L.b200lz4f_writer_free(self.h)


def _place(pieces, phases):
    """one source holding piece k at an offset = phases[k] (mod 16), 16 bytes at least between pieces"""
    offs, pos = [], 0
    for d, ph in zip(pieces, phases):
        pos = (pos + 15) // 16 * 16 + ph
        offs.append(pos)
        pos += len(d) + 16
    src = np.zeros(pos + 64, dtype=np.uint8)
    for o, d in zip(offs, pieces):
        src[o:o + len(d)] = np.frombuffer(d, dtype=np.uint8)
    return src, _u64(offs), _u64([len(d) for d in pieces])


def _drive(L, M, datas, bs_code, flags, cut, room, op=None, hc=0, known=None, phase=0, max_calls=200000, on_call=None):
    """every stream in one writer, one call per round until all are DONE: stream k's piece is cut(k, rest, status, need,
    left) bytes from where it stopped (left: what the last call did not take), placed at phase + position (mod 16), with
    room(k, status, need, room); op(k, covers_rest, status) (default: CLOSE once the piece covers the rest, else WRITE).  On
    every call the guards in front of, between and behind the ranges hold, produced <= room, need > 0 on MORE_*, a DONE
    stream takes and produces nothing.  -> (outputs, flush points per stream, calls)"""
    ns = len(datas)
    wr = _Writer(L, ns, bs_code, flags, hc, known)
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
        doff, q = [], 24
        for c in caps:
            doff.append(q)
            q += c + 24
        d_dst = M.full(q + 64, GUARD)
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


def _expected(b200, port, data, flushes, bs_code, flags, phase=0, known=None):
    """LZ4FrameOutputStream's frame for `data` with flush() at each offset of `flushes` (LZ4FrameOutputStream.java:178-306):
    blocks of blockMaxSize between flushes, a short one at each flush, each compressed by this library's fast block
    compressor at its phase, as the writer runs it"""
    flg = 0x60 | (0x10 if flags & 2 else 0) | (0x08 if flags & 4 else 0) | (0x04 if flags & 1 else 0)
    desc = bytes([flg, bs_code << 4]) + ((len(data) if known is None else known).to_bytes(8, "little") if flags & 4 else b"")
    out = bytearray(b"\x04\x22\x4d\x18" + desc + bytes([(port.xxh32(desc, 0) >> 8) & 0xFF]))
    bs = 1 << (8 + 2 * bs_code)
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
            stored = c <= 0 or c >= n
            payload = data[o:o + n] if stored else comp[co:co + c].tobytes()
            out += (len(payload) | (0x80000000 if stored else 0)).to_bytes(4, "little") + payload
            if flags & 2:
                out += port.xxh32(payload, 0).to_bytes(4, "little")
    out += bytes(4)
    if flags & 1:
        out += port.xxh32(data, 0).to_bytes(4, "little")
    return bytes(out)


def _compress_dev(L, M, datas, bs_code, flags, hc=0, phase=0):
    src, offs, lens = _place(datas, [phase] * len(datas))
    rc, d_dst, fo, fl = _write(L, M, M.up(src), offs, lens, bs_code, flags, hc)
    assert rc >= 0, rc
    out = M.down(d_dst)
    return [out[int(o):int(o) + int(n)].tobytes() for o, n in zip(fo, fl)]


def _read_back(b200, port, ref, frame, data):
    """the frame through the host reader, the incremental device reader (in two pieces), the restated reader and
    LZ4F_decompress where the reference library is built"""
    assert b200.decompress_frames(frame, len(data) + 8) == data
    assert port.frame_decompress(frame, len(data) + 8) == (len(data), data)
    if ref is not None:
        assert ref.frame_decompress(frame, len(data) + 8) == (len(data), data), "LZ4F_decompress"
    L, M = b200._native.lib(), _DevMem()
    rd = _Reader(L, 1, True)
    half = len(frame) // 2
    got, at = bytearray(), 0
    for piece, eof in ((frame[:half], False), (None, True)):
        piece = frame[at:] if piece is None else piece
        src = np.frombuffer(piece + bytes(16), dtype=np.uint8)
        room = len(data) + (4 << 20)                                        # any block's slot bound
        d_dst = M.full(room, GUARD)
        rc, st, used, prod, need = rd.read(M, M.up(src), _u64([0]), _u64([len(piece)]), [eof], d_dst, _u64([0]), _u64([room]))
        assert rc == 0
        got += M.down(d_dst)[:int(prod[0])].tobytes()
        at += int(used[0])
    rd.free()
    assert int(st[0]) == DONE and bytes(got) == data


def _cuts(rng):
    return {
        "whole": lambda k, rest, s, need, left: rest,
        "random": lambda k, rest, s, need, left: left + rng.randrange(0, 2 * need + 64) if s == MORE_INPUT else (left or rng.randrange(0, 300000)),
        "need": lambda k, rest, s, need, left: left + need if s == MORE_INPUT else (left if s == MORE_ROOM else 0),
        "need-1+1": lambda k, rest, s, need, left: left + (need + 1 if need == 1 else need - 1) if s == MORE_INPUT else (left if s == MORE_ROOM else 1),
        "drip": lambda k, rest, s, need, left: left + 1 if s == MORE_INPUT else (left if s == MORE_ROOM else 1),
    }


def _rooms(ample):
    return {
        "ample": lambda k, s, need, r: ample[k],
        "exact": lambda k, s, need, r: need if s == MORE_ROOM else r,
        "growing": lambda k, s, need, r: (2 * r + need // 3 + 1) if s == MORE_ROOM else r,
    }


def _datas(port):
    datas = _mixed(port)
    return [d for d in datas if len(d) <= 70000] if SIM else datas


def test_whole_content_parity(b200, port):
    """the mixed corpus, every bsCode and flags value (the emulator: a subset), cut at random, at need and at need -1 / +1,
    one byte at a time (short inputs) and whole, with ample, exact and growing room, each piece at the whole content's phase
    plus what was taken: every stream's output is b200lz4f_compress_dev's frame of the whole content"""
    L, M = b200._native.lib(), _DevMem()
    datas = _datas(port)
    combos = [(bs, fl) for bs in (4, 5, 6, 7) for fl in range(8)]
    if SIM:
        combos = [(4, 0), (4, 7), (5, 3), (7, 5)]
    rng = random.Random(3)
    cuts = _cuts(rng)
    names = ["whole", "random", "need", "need-1+1"]
    for ci, (bs, fl) in enumerate(combos):
        known = [len(d) for d in datas] if fl & 4 else None
        want = _compress_dev(L, M, datas, bs, fl, phase=5)
        ample = [L.b200lz4f_compress_bound(len(d), bs) for d in datas]
        rooms = _rooms(ample)
        for cn in (names[ci % 4], "whole") if ci < 4 else (names[ci % 4],):
            rn = [("ample", "exact", "growing")[(k + ci) % 3] for k in range(len(datas))]
            outs, _, _ = _drive(L, M, datas, bs, fl, cuts[cn], lambda k, *a: rooms[rn[k]](k, *a), known=known, phase=5)
            for k, (o, w) in enumerate(zip(outs, want)):
                assert bytes(o) == w, (bs, fl, cn, k, len(datas[k]))
    short = [d for d in datas if len(d) <= 100]
    for bs, fl in ((4, 7), (6, 1)):
        want = _compress_dev(L, M, short, bs, fl, phase=9)
        outs, _, _ = _drive(L, M, short, bs, fl, cuts["drip"], lambda k, s, need, r: need if s == MORE_ROOM else r,
                            known=[len(d) for d in short] if fl & 4 else None, phase=9)
        assert [bytes(o) for o in outs] == want


def test_flush_parity_and_every_reader(b200, port):
    """FLUSH at random points, FLUSH with an empty tail (twice in a row) and CLOSE right after a FLUSH: the output is the
    frame assembled by LZ4FrameOutputStream's rules, and it reads back through the host reader, the incremental reader, the
    restated reader and LZ4F_decompress"""
    L, M, ref = b200._native.lib(), _DevMem(), _reference()
    rng = random.Random(7)
    datas = [d for d in _datas(port) if len(d) <= (70000 if SIM else 1500000)]
    for bs, fl in (((4, 7), (5, 1)) if SIM else ((4, 7), (4, 0), (5, 3), (7, 5))):
        ample = [L.b200lz4f_compress_bound(len(d), bs) + 8 * (len(d) // 1000 + 8) for d in datas]
        rooms = _rooms(ample)
        ops = {}

        def op(k, covers, s):
            r = rng.random()
            o = (CLOSE if r < 0.5 else FLUSH) if covers else (FLUSH if r < 0.35 else WRITE)
            ops.setdefault(k, []).append(o)
            return o

        def cut(k, rest, s, need, left):
            return left + rng.choice([0, 1, 17, 1000, 70000, need or 1, rest])

        outs, flushes, _ = _drive(L, M, datas, bs, fl, cut, lambda k, *a: rooms[("ample", "growing")[k % 2]](k, *a), op=op,
                                  known=[len(d) for d in datas] if fl & 4 else None, phase=3)
        assert any(flushes)
        for k, (o, d) in enumerate(zip(outs, datas)):
            assert bytes(o) == _expected(b200, port, d, flushes[k], bs, fl, phase=3), (bs, fl, k, flushes[k])
            _read_back(b200, port, ref, bytes(o), d)


def test_high_compressor(b200, port):
    """hc_level 9, cut at random: the frames read back; on the emulator, where HC's order is fixed, they are
    b200lz4f_compress_dev's at the same level and phase (on the GPU the HC kernel's bucket ways are claimed with atomicAdd,
    so a block whose bucket wraps may parse differently from run to run)"""
    L, M, ref = b200._native.lib(), _DevMem(), _reference()
    datas = [port.datagen(n, 0.5, 0.0, 5 + n % 7).tobytes() for n in ((70000, 1) if SIM else (300000, 65537, 1, 0, 1500000))]
    want = _compress_dev(L, M, datas, 4, 7, hc=9, phase=0)
    rng = random.Random(2)
    outs, _, _ = _drive(L, M, datas, 4, 7, _cuts(rng)["random"], lambda k, s, need, r: 1 << 22, hc=9,
                        known=[len(d) for d in datas])
    for o, w, d in zip(outs, want, datas):
        _read_back(b200, port, ref, bytes(o), d)
        if SIM:
            assert bytes(o) == w


def test_latched_need_and_empty_frames(b200, port):
    """need on MORE_ROOM is the unit's bound (header 7 / 15, block 4 + len (+ 4), EndMark 4 / 8) and a call given exactly
    that progresses; need on MORE_INPUT is what the next whole block lacks, blockMaxSize after a flush.  A stream closed with
    no content is header + EndMark, compress_dev's frame of 0 bytes; DONE is latched; a known_size mismatch reads back -8"""
    L, M = b200._native.lib(), _DevMem()
    data = port.datagen(200000, 0.5, 0.0, 3).tobytes()

    def step(wr, piece, op, cap, at=0):
        src, offs, lens = _place([piece], [at % 16])
        d_dst = M.full(cap + 64, GUARD)
        rc, st, used, prod, need = wr.write(M, M.up(src), offs, lens, [op], d_dst, _u64([0]), _u64([cap]))
        out = M.down(d_dst)
        assert rc == 0 and (out[int(prod[0]):] == GUARD).all()
        return int(st[0]), int(used[0]), int(prod[0]), int(need[0]), out[:int(prod[0])].tobytes()

    for fl in (0, 7):
        wr = _Writer(L, 1, 4, fl, known=[len(data)] if fl & 4 else None)
        head, word, tail = 7 + (8 if fl & 4 else 0), 4 + (4 if fl & 2 else 0), 4 + (4 if fl & 1 else 0)
        got = bytearray()
        assert step(wr, data[:10], WRITE, head - 1)[:4] == (MORE_ROOM, 0, 0, head)
        s = step(wr, data[:10], WRITE, head)
        assert s[:4] == (MORE_INPUT, 0, head, 65536 - 10)
        got += s[4]
        assert step(wr, data[:65536 + 5], WRITE, 65536 + word - 1)[:4] == (MORE_ROOM, 0, 0, 65536 + word)
        s = step(wr, data[:65536 + 5], WRITE, 65536 + word)
        assert s[:2] == (MORE_INPUT, 65536) and s[3] == 65536 - 5
        got += s[4]
        assert step(wr, data[65536:65536 + 5], FLUSH, 5 + word - 1)[:4] == (MORE_ROOM, 0, 0, 5 + word)
        s = step(wr, data[65536:65536 + 5], FLUSH, 5 + word)
        assert s[:2] == (MORE_INPUT, 5) and s[3] == 65536
        got += s[4]
        assert step(wr, b"", FLUSH, 0)[:4] == (MORE_INPUT, 0, 0, 65536)            # an empty tail writes nothing
        s = step(wr, data[65541:65600], CLOSE, 59 + word + tail - 1, at=65541)     # the block fits, the EndMark does not
        assert s[:2] == (MORE_ROOM, 59) and s[3] == tail and s[2] <= 59 + word
        got += s[4]
        s = step(wr, b"", CLOSE, tail)                                             # the CLOSE repeated
        assert s[:4] == (DONE, 0, tail, 0)
        got += s[4]
        assert bytes(got) == _expected(b200, port, data[:65600], [65541], 4, fl, known=len(data))
        wr.free()
    # a stream closed with no content, and latching
    for fl in (0, 5):
        wr = _Writer(L, 1, 5, fl, known=[0] if fl & 4 else None)
        st, used, prod, need, out = step(wr, b"", CLOSE, 64)
        assert (st, used, need) == (DONE, 0, 0) and out == _compress_dev(L, M, [b""], 5, fl)[0]
        assert step(wr, data[:100], CLOSE, 1000) == (DONE, 0, 0, 0, b"")
        assert step(wr, data[:100], WRITE, 1000) == (DONE, 0, 0, 0, b"")
        wr.free()
    # a declared size that is not the content's: the writer does not check it, every reader answers -8
    wr = _Writer(L, 1, 4, 5, known=[len(data) + 1])
    st, used, prod, need, out = step(wr, data, CLOSE, 1 << 20)
    assert st == DONE and used == len(data)
    assert L.b200lz4f_decompress_host(out, len(out), np.empty(len(data) + 64, dtype=np.uint8).ctypes.data, len(data) + 64) == -8
    wr.free()


def test_many_streams_piped_into_the_reader(b200, port):
    """64 streams with mixed ops and pieces: each call's output goes straight to an incremental reader (what it does not take
    waits for the next call), and every stream's content comes back"""
    L, M = b200._native.lib(), _DevMem()
    rng = random.Random(13)
    base = port.datagen(1 << 20, 0.5, 0.0, 21).tobytes()
    ns = 64
    datas = [base[rng.randrange(0, 1000):][:rng.choice([0, 1, 500, 70000, 200000] if SIM else [0, 1, 500, 70000, 300000, 900000])]
             for _ in range(ns)]
    if SIM:
        datas = [d[:3000] for d in datas]
    rd = _Reader(L, ns, True)
    pending = [b""] * ns
    contents = [bytearray() for _ in range(ns)]
    rstat = [None] * ns

    def on_call(st, used, prod, dst, doff):
        for k in range(ns):
            pending[k] += dst[doff[k]:doff[k] + int(prod[k])].tobytes()
        src, offs, lens = _place(pending, [0] * ns)
        caps = [max(len(d), 65536) + 64 for d in datas]                     # a 64 KiB block's slot bound at least
        d_dst = M.full(sum(caps) + 64, GUARD)
        doffs = np.cumsum([0] + caps[:-1])
        rc, s, u, p, n = rd.read(M, M.up(src), offs, lens, [int(x) == DONE for x in st], d_dst, _u64(doffs), _u64(caps))
        assert rc == 0
        out = M.down(d_dst)
        for k in range(ns):
            contents[k] += out[int(doffs[k]):int(doffs[k]) + int(p[k])].tobytes()
            pending[k] = pending[k][int(u[k]):]
            rstat[k] = int(s[k])

    def op(k, covers, s):
        return CLOSE if covers else rng.choice([WRITE, WRITE, FLUSH])

    _drive(L, M, datas, 4, 7, lambda k, rest, s, need, left: left + rng.randrange(0, 150000),
           lambda k, s, need, r: rng.choice([need, 1 << 18]) if s == MORE_ROOM else r, op=op,
           known=[len(d) for d in datas], on_call=on_call)
    rd.free()
    assert rstat == [DONE] * ns
    assert [bytes(c) for c in contents] == datas


def test_errors_launch_nothing_and_write_nothing(b200, port):
    """create: bsCode 3 / 8, ns above 2^31 - 1, flags bit 2 without known sizes or with a negative one give NULL and
    B200LZ4_E_ARG.  write: a NULL writer or pointer, an op above CLOSE, a destination range that overflows give B200LZ4_E_ARG
    before anything is launched or written, and the stream's state is unchanged; a writer of 0 streams returns 0.  One
    stream of 64 blocks and 64 streams of one block launch the same kernels"""
    L, M = b200._native.lib(), _DevMem()
    err = ctypes.c_int(0)
    for args in ((1, 3, 0), (1, 8, 0), (1 << 31, 4, 0), (2, 4, 4)):
        assert not L.b200lz4f_writer_create(*args, 0, None, ctypes.byref(err)) and err.value == E_ARG, args
    neg = np.asarray([5, -1], dtype=np.int64)
    assert not L.b200lz4f_writer_create(2, 4, 4, 0, neg.ctypes.data, ctypes.byref(err)) and err.value == E_ARG
    data = port.datagen(100000, 0.5, 0.0, 6).tobytes()
    src, offs, lens = _place([data, b"xyz"], [0, 0])
    d_src, d_dst = M.up(src), M.full(300100, GUARD)
    doff, dcap = _u64([0, 200000]), _u64([150000, 100])
    wr = _Writer(L, 2, 4, 7, known=[len(data), 3])
    z = np.zeros(2, dtype=np.uint64)
    st = np.zeros(2, dtype=np.int32)
    ops = np.full(2, CLOSE, dtype=np.uint8)
    before = L.b200lz4_launch_count()
    args = [M.ptr(d_src), offs.ctypes.data, lens.ctypes.data, ops.ctypes.data, M.ptr(d_dst), doff.ctypes.data, dcap.ctypes.data,
            st.ctypes.data, z.ctypes.data, z.ctypes.data, z.ctypes.data, None]
    assert L.b200lz4f_writer_write_dev(None, *args) == E_ARG
    for i in range(11):
        bad = list(args)
        bad[i] = None
        assert L.b200lz4f_writer_write_dev(wr.h, *bad) == E_ARG, i
    bad = list(args)
    bad[3] = np.asarray([CLOSE, 3], dtype=np.uint8).ctypes.data
    assert L.b200lz4f_writer_write_dev(wr.h, *bad) == E_ARG
    bad = list(args)
    far = _u64([0, (1 << 64) - 50])
    bad[5] = far.ctypes.data
    assert L.b200lz4f_writer_write_dev(wr.h, *bad) == E_ARG
    assert L.b200lz4_launch_count() == before and (M.down(d_dst) == GUARD).all()
    empty = L.b200lz4f_writer_create(0, 4, 0, 0, None, ctypes.byref(err))
    assert empty and L.b200lz4f_writer_write_dev(empty, *([None] * 12)) == 0
    L.b200lz4f_writer_free(empty)
    rc, s, used, prod, need = wr.write(M, d_src, offs, lens, [CLOSE, CLOSE], d_dst, doff, dcap)
    assert rc == 0 and s.tolist() == [DONE, DONE] and used.tolist() == [len(data), 3]
    out = M.down(d_dst)
    assert out[:int(prod[0])].tobytes() == _compress_dev(L, M, [data], 4, 7)[0]
    wr.free()

    n = 8 if SIM else 64
    body = port.datagen(n * 65536, 0.5, 0.0, 7).tobytes()
    for fl in (0, 7):
        counts = []
        for datas in ([body], [body[k * 65536:(k + 1) * 65536] for k in range(n)]):
            src, offs, lens = _place(datas, [0] * len(datas))
            wr = _Writer(L, len(datas), 4, fl, known=[len(d) for d in datas] if fl & 4 else None)
            caps = [L.b200lz4f_compress_bound(len(d), 4) for d in datas]
            d_dst = M.full(sum(caps) + 64, 0)
            b = L.b200lz4_launch_count()
            rc, s, used, prod, need = wr.write(M, M.up(src), offs, lens, [CLOSE] * len(datas), d_dst, _u64(np.cumsum([0] + caps[:-1])), _u64(caps))
            counts.append(L.b200lz4_launch_count() - b)
            assert rc == 0 and (s == DONE).all()
            wr.free()
        assert counts[0] == counts[1], (fl, counts)


def _counted(L):
    if not hasattr(L, "b200lz4_sim_device_bytes"):
        pytest.skip("this emulator library does not count copies and allocations: tests/simt/alloc_count.h")
    L.b200lz4_sim_copied_bytes.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
    L.b200lz4_sim_device_bytes.argtypes = [ctypes.c_void_p, ctypes.c_void_p]


@pytest.mark.skipif(not SIM, reason="the counting emulator build counts the library's host<->device copies")
def test_per_call_copies_do_not_depend_on_payload(b200, port):
    """the same streams and block counts at block sizes 64 KiB and 256 KiB, with payloads of 1 and 3 blocks per call, at every
    flags value with a content checksum: every call copies the same bytes between host and device"""
    L, M = b200._native.lib(), _DevMem()
    _counted(L)
    h2d, d2h = ctypes.c_ulonglong(0), ctypes.c_ulonglong(0)
    counts = []
    for bs in (4, 5):
        size = 1 << (8 + 2 * bs)
        rng = random.Random(8)
        datas = [rng.randbytes(3 * size + 100) for _ in range(3)]
        wr = _Writer(L, len(datas), bs, 7, known=[len(d) for d in datas])
        pos = [0] * len(datas)
        for rnd, op in enumerate((WRITE, FLUSH, CLOSE)):
            pieces = [d[p:p + (size if rnd == 0 else 2 * size + (100 if op == CLOSE else 0))] for d, p in zip(datas, pos)]
            src, offs, lens = _place(pieces, [0] * len(pieces))
            caps = [4 * size] * len(datas)
            d_src, d_dst = M.up(src), M.full(sum(caps) + 64, 0)
            L.b200lz4_sim_copied_bytes(ctypes.byref(h2d), ctypes.byref(d2h))
            a = (h2d.value, d2h.value)
            rc, st, u, prod, need = wr.write(M, d_src, offs, lens, [op] * len(datas), d_dst, _u64(np.cumsum([0] + caps[:-1])), _u64(caps))
            L.b200lz4_sim_copied_bytes(ctypes.byref(h2d), ctypes.byref(d2h))
            counts.append((rnd, h2d.value - a[0], d2h.value - a[1]))
            pos = [p + int(x) for p, x in zip(pos, u)]
            assert rc == 0
        wr.free()
    assert counts[:3] == counts[3:], counts
    assert max(c[1] + c[2] for c in counts) < 4096, counts


@pytest.mark.skipif(not SIM, reason="the counting emulator build counts the library's device allocations")
def test_device_memory_does_not_grow_with_the_stream(b200, port):
    """one stream written 4 blocks per call: 16 blocks take less than 1 MiB of device scratch, and 64 blocks written behind
    them allocate nothing more"""
    L, M = b200._native.lib(), _DevMem()
    _counted(L)
    content = port.datagen(65536, 0.5, 0.0, 4).tobytes()
    grown = []
    for nblocks in (16, 64):
        live, peak = ctypes.c_ulonglong(0), ctypes.c_ulonglong(0)
        L.b200lz4_sim_reset_device_peak()
        L.b200lz4_sim_device_bytes(ctypes.byref(live), ctypes.byref(peak))
        base = live.value
        outs, _, calls = _drive(L, M, [content * nblocks], 4, 1, lambda k, rest, s, need, left: left + 4 * 65536,
                                lambda k, s, need, r: 4 * 65540 + 64)
        L.b200lz4_sim_device_bytes(ctypes.byref(live), ctypes.byref(peak))
        grown.append(peak.value - base)
        assert calls >= nblocks // 4 and b200.decompress_frames(bytes(outs[0]), 65536 * nblocks) == content * nblocks
    assert grown[0] < (1 << 20) and grown[1] == 0, grown


@pytest.mark.skipif(SIM, reason="device memory beyond the emulator's")
def test_frames_longer_than_the_card(b200, port):
    """one stream of 96 GiB of content at bsCode 4 with the content size declared: one 256 MiB device piece written again
    and again into one fixed output buffer, each call's output read at once by an incremental reader, so the frame never
    exists anywhere whole; the reader ends DONE with 96 GiB.  Then 5 GiB with a content checksum, past the 2 GiB that
    b200lz4f_compress_dev refuses: the reader ends DONE and the checksum word is the oracle's streaming XXH32 of the content"""
    import torch
    period = port.datagen(4 << 20, 0.5, 0.0, 17)
    piece = torch.from_numpy(period.copy()).cuda().repeat(64)                  # 256 MiB
    n = piece.numel()
    out = torch.empty(n + (n >> 16) * 8 + 64, dtype=torch.uint8, device="cuda")
    content = torch.empty(n, dtype=torch.uint8, device="cuda")

    def run(calls, checksum):
        total = calls * n
        wr = b200.FrameWriter(1, 4, content_checksum=checksum, known_size=total)
        rd = b200.FrameReader(1, read_single_frame=True)
        produced, last = 0, None
        for c in range(calls + 1):
            close = c == calls
            st, used, prod, need = wr.write(piece, [0], [0 if close else n], out, [0], [out.numel()], [CLOSE if close else WRITE])
            assert int(st[0]) == (DONE if close else MORE_INPUT) and int(used[0]) == (0 if close else n), (c, st, used)
            p = int(prod[0])
            rs, ru, rp, _ = rd.read(out, [0], [p], content, [0], [n], [close])
            assert int(ru[0]) == p and int(rs[0]) == (DONE if close else MORE_INPUT), (c, rs, ru, p)
            if not close:
                assert int(rp[0]) == n and bool(torch.equal(content, piece)), c
            produced += int(rp[0])
            last = out[p - 4:p].cpu().numpy().tobytes() if close else None
        wr.close()
        rd.close()
        return produced, last

    assert run(96 * 4, False)[0] == 96 << 30
    produced, last = run(5 * 4, True)
    assert produced == 5 << 30
    assert int.from_bytes(last, "little") == port.xxh_stream(32, [period.tobytes()] * (5 * 256))


@pytest.mark.skipif(SIM, reason="torch tensors and streams: GPU only")
def test_python_wrapper_and_stream_order(b200, port):
    """frame.FrameWriter against the C ABI, its argument checks, and a source written by a torch op on a side stream with
    the writer called on that stream without a synchronise: the frame holds the new bytes"""
    import torch
    L, M = b200._native.lib(), _DevMem()
    old, new = port.datagen(3 << 20, 0.5, 0.0, 1), port.datagen(3 << 20, 0.5, 0.0, 2)
    d_src, d_new = M.up(old), M.up(new)
    out = torch.full((8 << 20,), GUARD, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with b200.FrameWriter(2, 5, True, True, known_size=[3 << 19, 3 << 19]) as wr:
        with torch.cuda.stream(side):
            d_src.copy_(d_new)
            st, used, prod, need = wr.write(d_src, [0, 3 << 19], [3 << 19, 3 << 19], out, [0, 4 << 20], [4 << 20, 4 << 20],
                                            [b200.frame.CLOSE, b200.frame.WRITE])
        assert st.dtype == np.int32 and used.dtype == np.uint64 and prod.dtype == np.uint64 and need.dtype == np.uint64
        assert st.tolist() == [b200.frame.DONE, b200.frame.MORE_INPUT] and used.tolist() == [3 << 19, 3 << 19]
        st2, used2, prod2, _ = wr.write(d_src, [0, 0], [0, 0], out, [0, (4 << 20) + int(prod[1])], [0, 1 << 20],
                                        [b200.frame.CLOSE, b200.frame.CLOSE])
        assert st2.tolist() == [b200.frame.DONE, b200.frame.DONE] and prod2.tolist()[0] == 0
        host = out.cpu().numpy()
        f0 = host[:int(prod[0])].tobytes()
        f1 = host[4 << 20:(4 << 20) + int(prod[1]) + int(prod2[1])].tobytes()
        want = _compress_dev(L, M, [new[:3 << 19].tobytes(), new[3 << 19:].tobytes()], 5, 7)
        assert [f0, f1] == want
        assert (host[int(prod[0]):4 << 20] == GUARD).all()
        with pytest.raises(ValueError):
            wr.write(d_src, [0], [1], out, [0], [1], [0])                      # one entry, two streams
        with pytest.raises(ValueError):
            wr.write(d_src.cpu(), [0, 0], [1, 1], out, [0, 0], [1, 1], [0, 0])
        with pytest.raises(ValueError):
            wr.write(d_src, [0, 0], [1, 1], out, [0, 0], [1, (8 << 20) + 1], [0, 0])
        with pytest.raises(ValueError):
            wr.write(d_src, [0, 0], [1, 1], out, [0, 0], [1, 1], [0, 3])
    with pytest.raises(ValueError):
        wr.write(d_src, [0, 0], [1, 1], out, [0, 0], [1, 1], [0, 0])           # closed
    with pytest.raises(ValueError):
        b200.FrameWriter(1, 3)
    with pytest.raises(ValueError):
        b200.FrameWriter(1, 4, known_size=-1)
