"""b200lz4f_reader_*: the incremental device frame reader.  Each stream is one LZ4FrameInputStream(in, readSingleFrame) whose
bytes arrive in pieces; a call takes the complete units at the start of each piece and carries the stream's state to the
next call.  Whatever the pieces and the room, the concatenated content and the final status must be what the host reader
(b200lz4f_decompress_host / _single) gives for the whole stream, and on an error the content delivered in front of it must
be what a per-block restatement of readBlock delivers.  Runs on the H100, and on the CPU emulator build of the library
(B200LZ4_TEST_SO=.../libb200lz4_sim*.so), where the sizes shrink and torch is not used."""
import ctypes
import os
import random

import numpy as np
import pytest

from test_frame_decode_dev import SKIP, _frame_of_pieces
from test_frame_streams_dev import _cases, _host
from test_lz4block_dev import _DevMem, _lay_out, _u64

pytestmark = pytest.mark.gpu

SIM = "sim" in os.environ.get("B200LZ4_TEST_SO", "")
E_ARG = -2147483645
GUARD = 0xAA
MORE_INPUT, MORE_ROOM, DONE = 0, 1, 2
BIG = 1 << 23


def _u32(b, i):
    return int.from_bytes(b[i:i + 4], "little")


def _restate(port, blob, single):
    """LZ4FrameInputStream read block by block (readHeader / readBlock, the oracle's safe decoder and XXH32) -> (code or
    total, the content delivered before it stopped, where it stopped, the summed slot bounds of the blocks it read, a
    failing one included: room enough to read the whole stream in one call)"""
    out, ip, n, seen, bounds = bytearray(), 0, len(blob), False, 0
    fail = lambda code: (code, bytes(out), ip, bounds)
    while ip < n:
        if n - ip < 4:
            return fail(-1)
        magic = _u32(blob, ip)
        ip += 4
        if magic >> 4 == 0x184D2A5:
            if n - ip < 4:
                return fail(-1)
            sz = _u32(blob, ip)
            ip += 4
            if n - ip < sz:
                return fail(-1)
            ip += sz
            seen = True
            continue
        if magic != 0x184D2204:
            return fail(-2)
        d0 = ip
        if n - ip < 3:
            return fail(-1)
        flg, bd = blob[ip], blob[ip + 1]
        ip += 2
        if flg >> 6 != 1 or flg & 2 or not flg & 0x20 or flg & 1 or bd & 0x8F or bd >> 4 < 4:
            return fail(-10)
        bs = 1 << (8 + 2 * (bd >> 4))
        size = None
        if flg & 8:
            if n - ip < 9:
                return fail(-1)
            size = int.from_bytes(blob[ip:ip + 8], "little")
            ip += 8
        if n - ip < 1:
            return fail(-1)
        if (port.xxh32(blob[d0:ip], 0) >> 8) & 0xFF != blob[ip]:
            ip += 1
            return fail(-3)
        ip += 1
        frame = bytearray()
        while True:
            if n - ip < 4:
                return fail(-1)
            word = _u32(blob, ip)
            ip += 4
            sz = word & 0x7FFFFFFF
            if sz == 0:
                break
            if sz > bs:
                return fail(-4)
            if n - ip < sz:
                return fail(-1)
            payload = blob[ip:ip + sz]
            ip += sz
            bounds += sz if word >> 31 else min(bs, 255 * sz)                # the room the reader asks for this block
            if flg & 0x10:
                if n - ip < 4:
                    return fail(-1)
                if _u32(blob, ip) != port.xxh32(payload, 0):
                    return fail(-5)
                ip += 4
            if word >> 31:
                dec = payload
            else:
                r, dec = port.decompress_safe(payload, bs)
                if r < 0:
                    return fail(-6)
            out += dec
            frame += dec
        if flg & 4:
            if n - ip < 4:
                return fail(-1)
            want = _u32(blob, ip)
            ip += 4
            if port.xxh32(bytes(frame), 0) != want:
                return fail(-7)
        if size is not None and size != len(frame):
            return fail(-8)
        seen = True
        if single:
            break
    if not seen:
        return fail(-1)
    return len(out), bytes(out), ip, bounds


class _Reader:
    def __init__(self, L, ns, single):
        self.L, err = L, ctypes.c_int(0)
        self.h = L.b200lz4f_reader_create(ns, int(single), ctypes.byref(err))
        assert self.h and err.value == 0, err.value

    def read(self, M, d_src, offs, lens, eof, d_dst, doff, dcap, stream=None):
        ns = len(lens)
        st = np.zeros(ns, dtype=np.int32)
        used, prod, need = (np.zeros(ns, dtype=np.uint64) for _ in range(3))
        e = np.ascontiguousarray(np.asarray(eof, dtype=np.uint8))
        rc = self.L.b200lz4f_reader_read_dev(self.h, M.ptr(d_src), offs.ctypes.data, lens.ctypes.data, e.ctypes.data, M.ptr(d_dst),
                                             doff.ctypes.data, dcap.ctypes.data, st.ctypes.data, used.ctypes.data,
                                             prod.ctypes.data, need.ctypes.data, stream)
        return rc, st, used, prod, need

    def free(self):
        self.L.b200lz4f_reader_free(self.h)


def _drive(L, M, blobs, single, cut, room, max_calls=100000, extra=1):
    """every stream in one reader, one call per round: stream k's piece is cut(k, rest, status, need, piece) bytes from where it
    stopped, its room room(k, status, need, room).  Each call's guard bytes around and behind each stream's produced range
    must be untouched, a latched stream must take and produce nothing.  -> (status, content, consumed, calls)"""
    ns = len(blobs)
    rd = _Reader(L, ns, single)
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
        doff, p = [], 24
        for c in caps:
            doff.append(p)
            p += c + 24
        doff = _u64(doff)
        d_dst = M.full(p + 64, GUARD)
        rc, st, used, prod, nd = rd.read(M, M.up(src), offs, lens, eof, d_dst, doff, _u64(caps))
        assert rc == 0, rc
        calls += 1
        dst = M.down(d_dst)
        assert (dst[:24] == GUARD).all()
        for k in range(ns):
            s, u, pr = int(st[k]), int(used[k]), int(prod[k])
            if status[k] is not None and (status[k] < 0 or status[k] == DONE):
                assert s == status[k] and u == 0 and pr == 0, (k, s, status[k], u, pr)
            assert u <= piece[k] and pr <= caps[k], (k, u, piece[k], pr, caps[k])
            o = int(doff[k])
            assert (dst[o + pr:o + caps[k] + 24] == GUARD).all(), (k, s, pr, caps[k])
            outs[k] += dst[o:o + pr].tobytes()
            pos[k] += u
            status[k], need[k] = s, int(nd[k])
            if s in (MORE_INPUT, MORE_ROOM):
                assert need[k] > 0, (k, s)
        assert calls <= max_calls, (calls, status)
    rd.free()
    return status, outs, pos, calls


def _check(L, port, blobs, single, status, outs, pos, seen=None):
    for k, b in enumerate(blobs):
        want, h_used, h_out = _host(L, b, BIG, single)
        code, delivered, _, _ = _restate(port, b, single)
        assert code == want, (k, code, want)
        if want >= 0:
            assert status[k] == DONE and outs[k] == h_out and pos[k] == h_used, (single, k, status[k], len(outs[k]), want, pos[k], h_used)
        else:
            assert status[k] == want and outs[k] == delivered, (single, k, status[k], want, len(outs[k]), len(delivered))
        if seen is not None:
            seen[want if want < 0 else "ok"] = seen.get(want if want < 0 else "ok", 0) + 1


# cut schedules: how many bytes of the rest to present, from where the stream stopped
def _cuts(rng):
    return {
        "whole": lambda k, rest, s, need, p: rest,
        "random": lambda k, rest, s, need, p: need + rng.randrange(0, 2 * need + 64) if s == MORE_INPUT else rng.randrange(0, 200),
        "need": lambda k, rest, s, need, p: need if s == MORE_INPUT else (p - 0 if s == MORE_ROOM else 0),
        "need-1+1": lambda k, rest, s, need, p: (need + 1 if p == need - 1 else need - 1) if s == MORE_INPUT else (p if s == MORE_ROOM else 1),
        "drip": lambda k, rest, s, need, p: p + 1 if s == MORE_INPUT else (p if s == MORE_ROOM else 1),
    }


# room schedules
def _rooms(ample):
    return {
        "ample": lambda k, s, need, r: ample[k] + 16,
        "exact": lambda k, s, need, r: need if s == MORE_ROOM else r,
        "growing": lambda k, s, need, r: (2 * r + need // 3 + 1) if s == MORE_ROOM else r,
    }


def _parity(b200, port, single, cut_names, room_names, short_only=False, n=None):
    L, M = b200._native.lib(), _DevMem()
    rng = random.Random(31 + single)
    blobs = _cases(b200, port, rng, (n if n is not None else (6 if SIM else 80)))
    if short_only:
        blobs = [b for b in blobs if len(b) <= (160 if SIM else 3000)]
    ample = [_restate(port, b, single)[3] for b in blobs]
    cuts, rooms = _cuts(random.Random(5)), _rooms(ample)
    seen = {}
    for ci, cn in enumerate(cut_names):
        rn = [room_names[(k + ci) % len(room_names)] for k in range(len(blobs))]
        status, outs, pos, _ = _drive(L, M, blobs, single, lambda k, *a: cuts[cn](k, *a), lambda k, *a: rooms[rn[k]](k, *a), extra=2)
        _check(L, port, blobs, single, status, outs, pos, seen)
    return seen


@pytest.mark.parametrize("single", [False, True])
def test_split_parity_on_faulty_streams(b200, port, single):
    """the streams of test_frame_streams_dev (faulty, flushed, skippable, empty, every bsCode and flags value) read whole,
    cut at random past each unit, cut at exactly need and at need -1 / +1 (the emulator: the last only), all in one reader per
    schedule, with ample, exact
    and growing-from-zero room spread over the streams: status, content and total consumed are the host reader's; on an
    error the content delivered is the restated reader's; guards hold on every call and latched streams stay put"""
    cuts = ["need-1+1"] if SIM else ["whole", "random", "need", "need-1+1"]
    seen = _parity(b200, port, single, cuts, ["ample", "exact", "growing"])
    want = {"ok", -1, -3} | (set() if single else {-2})                     # the corpus's -2 lies behind a first frame
    assert want <= set(seen) and len([k for k in seen if k != "ok"]) >= (3 if SIM else 5), seen


@pytest.mark.parametrize("single", [False, True])
def test_split_parity_one_byte_drip(b200, port, single):
    """the short streams of the same corpus fed one byte more per call"""
    _parity(b200, port, single, ["drip"], ["exact", "growing"], short_only=True)


def test_progress_bound(b200, port):
    """a driver that presents the whole rest and grows the room to need on MORE_ROOM, from 0: every valid stream finishes in
    at most its unit count + 3 calls"""
    L, M = b200._native.lib(), _DevMem()
    data = port.datagen(1 << 18, 0.5, 0.0, 12).tobytes()
    blobs = [_frame_of_pieces(port, [data[k * 997:k * 997 + n] for k, n in enumerate((5000, 17, 65536, 100, 3000))], 4, block_checksum=True),
             SKIP + b200.compress_frame(data[:200000], 4, True, True, True) + SKIP,
             b200.compress_frame(data[:70000], 5, False, False, False), SKIP * 3]
    units = []
    for b in blobs:
        ip, u = 0, 0
        while ip < len(b):
            if _u32(b, ip) >> 4 == 0x184D2A5:
                ip += 8 + _u32(b, ip + 4)
                u += 2
                continue
            flg = b[ip + 4]
            ip += 7 + (8 if flg & 8 else 0)
            u += 1
            while True:
                sz = _u32(b, ip) & 0x7FFFFFFF
                ip += 4
                u += 1
                if sz == 0:
                    ip += 4 if flg & 4 else 0
                    break
                ip += sz + (4 if flg & 0x10 else 0)
        units.append(u)
    for k, b in enumerate(blobs):
        status, outs, pos, calls = _drive(L, M, [b], False, lambda k_, rest, s, need, p: rest,
                                          lambda k_, s, need, r: need if s == MORE_ROOM else r, extra=0)
        want, used, content = _host(L, b, BIG, False)
        assert status[0] == DONE and outs[0] == content and pos[0] == used
        assert calls <= units[k] + 3, (k, calls, units[k])


def test_latched_and_need(b200, port):
    """need for MORE_INPUT: 4 for a magic, 5 for a header's FLG, the header length, 8 for a skippable header, the whole block
    (word, payload, checksum), 8 for an EndMark with a content checksum; need for MORE_ROOM: the block's slot bound.  Room 0
    writes nothing.  DONE and errors are latched"""
    L, M = b200._native.lib(), _DevMem()
    data = port.datagen(100000, 0.5, 0.0, 3).tobytes()
    f = _frame_of_pieces(port, [data[:5000], data[:300]], 4, content_checksum=True, block_checksum=True, stored={1})
    c0 = _u32(f, 7) & 0x7FFFFFFF
    rd = _Reader(L, 1, False)

    def step(piece, cap, eof=False):
        src, offs, lens = _lay_out([piece])
        d_dst = M.full(cap + 64, GUARD)
        rc, st, used, prod, need = rd.read(M, M.up(src), offs, lens, [eof], d_dst, _u64([0]), _u64([cap]))
        out = M.down(d_dst)
        assert rc == 0 and (out[int(prod[0]):] == GUARD).all()
        return int(st[0]), int(used[0]), int(prod[0]), int(need[0]), out[:int(prod[0])].tobytes()

    assert step(b"", 0) == (MORE_INPUT, 0, 0, 4, b"")
    assert step(f[:4], 0) == (MORE_INPUT, 0, 0, 5, b"")
    assert step(f[:6], 0) == (MORE_INPUT, 0, 0, 7, b"")
    assert step(f[:7 + 3], 0) == (MORE_INPUT, 7, 0, 4, b"")                  # the header is taken alone
    rest = f[7:]
    assert step(rest[:6], 0) == (MORE_INPUT, 0, 0, 4 + c0 + 4, b"")
    assert step(rest[:8 + c0], 0) == (MORE_ROOM, 0, 0, min(65536, 255 * c0), b"")
    st, used, prod, need, out = step(rest, 65536)
    assert (st, used, prod, need) == (MORE_ROOM, 8 + c0, 5000, 300) and out == data[:5000]
    rest = rest[used:]
    st, used, prod, need, out = step(rest[:-1], 300)
    assert (st, used, prod, need) == (MORE_INPUT, 308, 300, 8) and out == data[:300]
    rest = rest[used:]
    assert step(rest, 0, eof=True) == (DONE, 8, 0, 0, b"")
    assert step(b"xyz", 100, eof=True) == (DONE, 0, 0, 0, b"")
    rd.free()
    rd = _Reader(L, 1, False)
    assert step(SKIP[:5], 0) == (MORE_INPUT, 0, 0, 8, b"")
    assert step(SKIP[:9], 0) == (MORE_INPUT, 9, 0, 2, b"")                  # a skippable payload in portions
    assert step(SKIP[9:], 0, eof=True) == (DONE, 2, 0, 0, b"")               # skippable frames only, as for the host reader
    assert step(f, 1 << 20, eof=True) == (DONE, 0, 0, 0, b"")
    rd.free()
    rd = _Reader(L, 1, False)
    assert step(b"", 0, eof=True) == (-1, 0, 0, 0, b"")                      # no frame at all
    assert step(f, 1 << 20, eof=True) == (-1, 0, 0, 0, b"")
    rd.free()


def test_errors_launch_nothing_and_write_nothing(b200, port):
    """a NULL reader or pointer, a destination range that overflows: B200LZ4_E_ARG before anything is launched, nothing
    written, the state unchanged; a reader of 0 streams: 0; ns above 2^31 - 1: no reader"""
    L, M = b200._native.lib(), _DevMem()
    frame = b200.compress_frame(port.datagen(100000, 0.5, 0.0, 6).tobytes(), 4, True, False, False)
    src, offs, lens = _lay_out([frame, b"xyz"])
    d_src, d_dst = M.up(src), M.full(300100, GUARD)
    doff, dcap = _u64([0, 300000]), _u64([200000, 3])                       # room for both blocks' slot bounds
    rd = _Reader(L, 2, False)
    z = np.zeros(2, dtype=np.uint64)
    st = np.zeros(2, dtype=np.int32)
    e = np.ones(2, dtype=np.uint8)
    before = L.b200lz4_launch_count()
    args = [M.ptr(d_src), offs.ctypes.data, lens.ctypes.data, e.ctypes.data, M.ptr(d_dst), doff.ctypes.data, dcap.ctypes.data,
            st.ctypes.data, z.ctypes.data, z.ctypes.data, z.ctypes.data, None]
    assert L.b200lz4f_reader_read_dev(None, *args) == E_ARG
    for i in (0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10):
        bad = list(args)
        bad[i] = None
        assert L.b200lz4f_reader_read_dev(rd.h, *bad) == E_ARG, i
    bad = list(args)
    far = _u64([0, (1 << 64) - 2])
    bad[5] = far.ctypes.data
    assert L.b200lz4f_reader_read_dev(rd.h, *bad) == E_ARG
    assert L.b200lz4_launch_count() == before and (M.down(d_dst) == GUARD).all()
    err = ctypes.c_int(0)
    assert not L.b200lz4f_reader_create(1 << 31, 0, ctypes.byref(err)) and err.value == E_ARG
    empty = L.b200lz4f_reader_create(0, 0, ctypes.byref(err))
    assert empty and L.b200lz4f_reader_read_dev(empty, *([None] * 11 + [None])) == 0
    L.b200lz4f_reader_free(empty)
    rc, s, used, prod, need = rd.read(M, d_src, offs, lens, [1, 1], d_dst, doff, dcap)
    assert rc == 0 and s.tolist() == [DONE, -1] and used.tolist()[0] == len(frame) and prod.tolist() == [100000, 0]
    rd.free()


def test_launches_do_not_depend_on_streams_frames_or_blocks(b200, port):
    """the same bytes as 1, 4 and 16 one-frame streams, and one 16-block frame against 16 one-block frames, each read in two
    calls (all but the last 6 bytes, then the rest): each of the two calls launches the same kernels whatever the split"""
    L, M = b200._native.lib(), _DevMem()
    m = 16
    data = port.datagen(m * 65536, 0.5, 0.0, 7).tobytes()
    counts = []

    def run(blobs, caps):
        rd = _Reader(L, len(blobs), False)
        out, used, calls = [], [len(b) - 8 for b in blobs], []            # in front of the EndMark and content checksum
        for first in (True, False):
            pieces = [b[:u + 2] if first else b[u:] for b, u in zip(blobs, used)]
            src, offs, lens = _lay_out(pieces)
            doff = _u64(np.cumsum(caps) - caps)
            d_dst = M.full(int(sum(caps)) + 64, GUARD)
            before = L.b200lz4_launch_count()
            rc, st, u, prod, need = rd.read(M, M.up(src), offs, lens, [not first] * len(blobs), d_dst, doff, _u64(caps))
            calls.append(L.b200lz4_launch_count() - before)
            assert rc == 0 and (st == (MORE_INPUT if first else DONE)).all(), st
            assert (u == (_u64(used) if first else lens)).all(), (u, lens)
            dst = M.down(d_dst)
            out.append([dst[int(o):int(o) + int(p)].tobytes() for o, p in zip(doff, prod)])
        counts.append(tuple(calls))
        rd.free()
        return [a + b for a, b in zip(*out)]

    for ns in (1, 4, 16):
        per = len(data) // ns
        blobs = [_frame_of_pieces(port, [data[j * 65536:(j + 1) * 65536] for j in range(k * m // ns, (k + 1) * m // ns)], 4,
                                  block_checksum=True) for k in range(ns)]
        got = run(blobs, [per] * ns)
        assert b"".join(got) == data
    one = _frame_of_pieces(port, [data[k * 65536:(k + 1) * 65536] for k in range(m)], 4, block_checksum=True)
    many = [_frame_of_pieces(port, [data[k * 65536:(k + 1) * 65536]], 4, block_checksum=True) for k in range(m)]
    assert b"".join(run([one], [m * 65536])) == data
    assert b"".join(run(many, [65536] * m)) == data
    assert len(set(counts)) == 1, counts


def _counted(L):
    if not hasattr(L, "b200lz4_sim_device_bytes"):
        pytest.skip("this emulator library does not count copies and allocations: tests/simt/alloc_count.h")
    L.b200lz4_sim_copied_bytes.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
    L.b200lz4_sim_device_bytes.argtypes = [ctypes.c_void_p, ctypes.c_void_p]


@pytest.mark.skipif(not SIM, reason="the counting emulator build counts the library's host<->device copies")
def test_per_call_copies_do_not_depend_on_payload(b200, port):
    """the same streams and frames with payloads 16x apart, read in two calls each: every call copies the same bytes
    between host and device, the per-stream arguments, states and results and a few totals"""
    L, M = b200._native.lib(), _DevMem()
    _counted(L)
    h2d, d2h = ctypes.c_ulonglong(0), ctypes.c_ulonglong(0)
    rng = random.Random(8)
    counts = []
    for size in (4096, 65536):
        frame = lambda: _frame_of_pieces(port, [rng.randbytes(size) for _ in range(4)], 4, block_checksum=True, stored=set(range(4)))
        blobs = [frame(), SKIP + frame() + SKIP, frame() + frame(), frame()[:-3]]
        rd = _Reader(L, len(blobs), False)
        used = [0] * len(blobs)
        for first in (True, False):
            pieces = [b[:len(b) // 2] if first else b[u:] for b, u in zip(blobs, used)]
            src, offs, lens = _lay_out(pieces)
            caps = _u64([8 * size] * len(blobs))
            doff = _u64(np.cumsum(caps) - caps)
            d_src, d_dst = M.up(src), M.full(int(sum(caps)) + 64, 0)
            L.b200lz4_sim_copied_bytes(ctypes.byref(h2d), ctypes.byref(d2h))
            a = (h2d.value, d2h.value)
            rc, st, u, prod, need = rd.read(M, d_src, offs, lens, [not first] * len(blobs), d_dst, doff, caps)
            L.b200lz4_sim_copied_bytes(ctypes.byref(h2d), ctypes.byref(d2h))
            counts.append((h2d.value - a[0], d2h.value - a[1]))
            used = [x + int(y) for x, y in zip(used, u)] if first else used
            assert rc == 0 and st.tolist() == ([MORE_INPUT] * 4 if first else [DONE, DONE, DONE, -1]), st
        rd.free()
    assert len(set(counts)) == 1, counts
    assert sum(counts[0]) < 4 * 600 + 1024, counts


@pytest.mark.skipif(not SIM, reason="the counting emulator build counts the library's device allocations")
def test_device_memory_does_not_grow_with_the_stream(b200, port):
    """one frame of one 64 KiB block repeated, fed in pieces of 4 blocks: a stream of 16 blocks takes less than 1 MiB of device
    scratch, and one of 64 blocks read behind it allocates nothing more"""
    L, M = b200._native.lib(), _DevMem()
    _counted(L)
    content = port.datagen(65536, 0.5, 0.0, 4).tobytes()
    block = _frame_of_pieces(port, [content], 4, content_checksum=False)[7:-4]
    head = bytes(_frame_of_pieces(port, [b"x"], 4, content_checksum=True)[:7])
    grown = []
    for nblocks in (16, 64):
        frame = head + block * nblocks + bytes(4) + port.xxh_stream(32, [content] * nblocks).to_bytes(4, "little")
        live, peak = ctypes.c_ulonglong(0), ctypes.c_ulonglong(0)
        L.b200lz4_sim_reset_device_peak()
        L.b200lz4_sim_device_bytes(ctypes.byref(live), ctypes.byref(peak))
        base = live.value
        status, outs, pos, calls = _drive(L, M, [frame], False, lambda k, rest, s, need, p: 4 * len(block) + 7,
                                          lambda k, s, need, r: 4 * 65536, extra=0)
        assert status[0] == DONE and outs[0] == content * nblocks and calls >= nblocks // 4
        L.b200lz4_sim_device_bytes(ctypes.byref(live), ctypes.byref(peak))
        grown.append(peak.value - base)
    assert grown[0] < (1 << 20) and grown[1] == 0, grown


@pytest.mark.skipif(SIM, reason="device memory beyond the emulator's")
def test_frames_longer_than_the_card(b200, port):
    """one frame of 96 GiB of content (bsCode 7, content size declared, no content checksum), one compressed 4 MiB block
    repeated, fed in 256 MiB pieces: every piece's content is the repeated block and the stream ends DONE.  Then 5 GiB with a
    content checksum from the oracle's streaming XXH32: clean, and with one flipped checksum bit -7 after all its content"""
    import torch
    L = b200._native.lib()
    bs = 4 << 20
    content = port.datagen(bs, 0.5, 0.0, 17).tobytes()
    one = b200.compress_frame(content, 7, False, False, False)               # header 7, one block, EndMark
    block = one[7:-4]
    assert len(block) < bs and _u32(block, 0) == len(block) - 4
    d_block = torch.from_numpy(np.frombuffer(content, dtype=np.uint8).copy()).cuda()
    piece_bytes = 256 << 20
    per = piece_bytes // len(block)                                          # whole blocks per piece
    body = torch.from_numpy(np.frombuffer(block, dtype=np.uint8).copy()).cuda().repeat(per)
    out = torch.empty(per * bs, dtype=torch.uint8, device="cuda")

    def header(flg, size):
        d = bytes([flg, 7 << 4]) + (size.to_bytes(8, "little") if flg & 8 else b"")
        return b"\x04\x22\x4d\x18" + d + bytes([(port.xxh32(d, 0) >> 8) & 0xFF])

    def read(nblocks, flg, tail):
        rd = b200.FrameReader(1)
        head = torch.from_numpy(np.frombuffer(header(flg, nblocks * bs), dtype=np.uint8).copy()).cuda()
        st, _, _, _ = rd.read(head, [0], [len(head)], out, [0], [0], [False])
        assert st.tolist() == [MORE_INPUT]
        left, produced, status = nblocks, 0, None
        while True:
            k = min(left, per)
            if k == per and left > per:
                src, eof = body, False
            else:                                                            # the last piece: its blocks and the EndMark
                src, eof = torch.cat([body[:k * len(block)], torch.from_numpy(np.frombuffer(tail, dtype=np.uint8).copy()).cuda()]), True
            st, used, prod, need = rd.read(src, [0], [src.numel()], out, [0], [per * bs], [eof])
            p = int(prod[0])
            assert p == k * bs and int(used[0]) == k * len(block) + (len(tail) if st[0] == DONE else 0), (st, used, prod, k)
            assert bool((out[:p].view(k, bs) == d_block).all())
            produced += p
            left -= k
            status = int(st[0])
            if status != MORE_INPUT:
                break
        rd.close()
        return status, produced

    assert read(96 * 256, 0x68, bytes(4)) == (DONE, 96 << 30)
    n5 = 5 * 256
    h = port.xxh_stream(32, [content] * n5)
    assert read(n5, 0x64, bytes(4) + h.to_bytes(4, "little")) == (DONE, 5 << 30)
    assert read(n5, 0x64, bytes(4) + (h ^ 0x100).to_bytes(4, "little")) == (-7, 5 << 30)


@pytest.mark.skipif(SIM, reason="torch tensors: GPU only")
def test_python_wrapper(b200, port):
    import torch
    data = port.datagen(300003, 0.5, 0.0, 9)
    src = torch.from_numpy(data.copy()).cuda()
    frames, fo, fl = b200.compress_frames_dev(src, [0, 300000], [300000, 3], 5, True, True, True)
    out = torch.full((1 << 20,), GUARD, dtype=torch.uint8, device="cuda")
    with b200.FrameReader(2) as rd:
        half = int(fl[0]) // 2
        st, used, prod, need = rd.read(frames, [int(fo[0]), int(fo[1])], [half, int(fl[1])], out, [0, 700000], [600000, 3],
                                       [False, True])
        assert st.dtype == np.int32 and used.dtype == np.uint64 and prod.dtype == np.uint64 and need.dtype == np.uint64
        assert st.tolist() == [b200.frame.MORE_INPUT, b200.frame.DONE] and used.tolist()[1] == int(fl[1]) and prod.tolist()[1] == 3
        p0 = int(prod[0])
        st2, used2, prod2, _ = rd.read(frames, [int(fo[0]) + int(used[0]), 0], [int(fl[0]) - int(used[0]), 0], out, [p0, 700000],
                                       [600000 - p0, 3], [True, True])
        assert st2.tolist() == [b200.frame.DONE, b200.frame.DONE] and prod2.tolist() == [300000 - p0, 0]
        host = out.cpu().numpy()
        assert host[:300000].tobytes() == data[:300000].tobytes() and host[700000:700003].tobytes() == data[300000:].tobytes()
        assert (host[300000:700000] == GUARD).all()
        with pytest.raises(ValueError):
            rd.read(frames, [0], [1], out, [0], [1], [True])                 # one entry, two streams
        with pytest.raises(ValueError):
            rd.read(frames.cpu(), [0, 0], [1, 1], out, [0, 0], [1, 1], [True, True])
        with pytest.raises(ValueError):
            rd.read(frames, [0, 0], [1, 1], out, [0, 0], [1, (1 << 20) + 1], [True, True])
    with pytest.raises(ValueError):
        rd.read(frames, [0, 0], [1, 1], out, [0, 0], [1, 1], [True, True])   # closed
