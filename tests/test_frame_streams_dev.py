"""b200lz4f_decompress_streams_dev: many independent LZ4 frame streams in device memory, each read as its own
LZ4FrameInputStream(in, readSingleFrame) into device memory, one result per stream.  Every stream's result, src_consumed and
content must be what the host reader (b200lz4f_decompress_host / _single) and the restated LZ4FrameInputStream give for that
stream alone.  Runs on the H100, and on the CPU emulator build of the library (B200LZ4_TEST_SO=.../libb200lz4_sim.so), where
the sizes shrink and torch is not used."""
import ctypes
import os
import random

import numpy as np
import pytest

from test_frame_decode_dev import SKIP, _datas, _faulty, _frame_of_pieces
from test_lz4block_dev import _DevMem, _lay_out, _u64

pytestmark = pytest.mark.gpu

SIM = "sim" in os.environ.get("B200LZ4_TEST_SO", "")
E_ARG = -2147483645
GUARD = 0xAA
BIG = 1 << 23


def _read(L, M, d_src, offs, lens, d_dst, doff, dcap, single, stream=None, result=True):
    """one b200lz4f_decompress_streams_dev call -> (rc, result, src_consumed, content_len)"""
    ns = len(lens)
    res, used, content = np.zeros(ns, dtype=np.int64), np.zeros(ns, dtype=np.uint64), np.zeros(ns, dtype=np.uint64)
    rc = L.b200lz4f_decompress_streams_dev(M.ptr(d_src), offs.ctypes.data, lens.ctypes.data, ns, M.ptr(d_dst), doff.ctypes.data,
                                           dcap.ctypes.data, int(single), res.ctypes.data if result else None, used.ctypes.data,
                                           content.ctypes.data, stream)
    return rc, res, used, content


def _host(L, blob, cap, single):
    """b200lz4f_decompress_host / _single on one stream -> (result, src_consumed (0 unless result >= 0), bytes)"""
    src = np.frombuffer(bytes(blob) + bytes(64), dtype=np.uint8)
    dst = np.zeros(max(cap, 1), dtype=np.uint8)
    if single:
        used = ctypes.c_size_t(0)
        r = L.b200lz4f_decompress_host_single(src.ctypes.data, len(blob), dst.ctypes.data, cap, ctypes.byref(used))
        used = used.value
    else:
        r = L.b200lz4f_decompress_host(src.ctypes.data, len(blob), dst.ctypes.data, cap)
        used = len(blob)                                            # the reader reads a whole container to its end
    return r, (used if r >= 0 else 0), dst[:max(r, 0)].tobytes()


def _dst_ranges(caps, order=None, slack=24):
    """destination offsets with `slack` guard bytes before, between and after the ranges, laid out in `order`"""
    order = range(len(caps)) if order is None else order
    doff, pos = [0] * len(caps), slack
    for k in order:
        doff[k] = pos
        pos += int(caps[k]) + slack
    return _u64(doff), pos + 64


def _read_all(L, M, blobs, caps, single, order=None):
    """every stream in ONE call, sources at phase 3 with gaps, destinations with guard bytes -> (res, used, content, dst, doff)"""
    src, offs, lens = _lay_out(blobs, align=16, phase=3, gap=5)
    doff, size = _dst_ranges(caps, order)
    d_src, d_dst = M.up(src), M.full(size, GUARD)
    rc, res, used, content = _read(L, M, d_src, offs, lens, d_dst, doff, _u64(caps), single)
    assert rc == 0, rc
    return res, used, content, M.down(d_dst), doff


def _check(L, port, blobs, caps, single, res, used, content, dst, doff, seen=None):
    """stream by stream against the host reader alone (and the restated reader when single is off); guard bytes untouched"""
    for k, (blob, cap) in enumerate(zip(blobs, caps)):
        want, h_used, h_out = _host(L, blob, cap, single)
        full, _, f_out = _host(L, blob, BIG, single)
        if not single:                      # the restated reader meets -9 where it happens, so it is asked with ample room
            assert port.frame_decompress(blob, BIG) == (full, f_out), (k, full)
        assert int(res[k]) == want and int(used[k]) == h_used, (single, k, int(res[k]), want, int(used[k]), h_used)
        got = dst[doff[k]:doff[k] + cap]
        if want >= 0:
            assert int(content[k]) == want and got[:want].tobytes() == h_out, (single, k)
            assert (got[want:] == GUARD).all(), (single, k)
        else:
            assert (got == GUARD).all(), (single, k, want)                  # a failing stream writes nothing
            assert int(content[k]) == (full if want == -9 else 0), (single, k, want, full, int(content[k]))
        assert (dst[doff[k] + cap:doff[k] + cap + 24] == GUARD).all(), (single, k)
        if seen is not None:
            seen[want if want < 0 else "ok"] = seen.get(want if want < 0 else "ok", 0) + 1
    assert (dst[:doff[0]] == GUARD).all()


def _cases(b200, port, rng, n):
    """faulty streams of either writer, flushed frames, skippable frames around and between frames, streams of skippable
    frames only, empty streams, and frames of every bsCode and flags"""
    base = port.datagen(1 << 18, 0.5, 0.0, 21).tobytes()
    blobs = [_faulty(rng, port, base) for _ in range(n)]
    flushed = []
    for trial in range(3 if SIM else 8):
        sizes = [rng.choice((1, 5, 16, 17, 100, 4097, 65535, 65536)) for _ in range(rng.randrange(1, 6 if SIM else 20))]
        pieces = [base[o:o + k] for o, k in ((rng.randrange(0, 100000), k) for k in sizes)]
        flushed.append(_frame_of_pieces(port, pieces, rng.choice((4, 5, 6, 7)), content_checksum=trial % 3 != 2,
                                        block_checksum=bool(trial & 1), stored={i for i in range(len(pieces)) if rng.random() < 0.15}))
    plain = b200.compress_frame(base[:150000], 4, True, True, False)
    blobs += flushed
    blobs += [SKIP + flushed[0] + SKIP + plain + SKIP, SKIP + plain, plain + SKIP + SKIP, SKIP, SKIP * 3, b"", b"",
              plain + flushed[1] + plain, SKIP + plain + b"\x00garbage that is not a frame", plain[:-1], b"\x04\x22\x4d",
              plain[:6] + bytes([plain[6] ^ 1]) + plain[7:]]                  # its header checksum byte
    combos = [(bs, fl) for bs in (4, 5, 6, 7) for fl in range(8)]
    if SIM:
        combos = [(4, 0), (4, 7), (5, 3), (6, 5), (7, 6)]
    for bs, fl in combos:
        d = base[:rng.choice((0, 1, 1000, 70000))]
        blobs.append(b200.compress_frame(d, bs, bool(fl & 1), bool(fl & 2), bool(fl & 4)))
    return blobs


def test_parity_on_faulty_streams_in_one_call(b200, port):
    """hundreds of streams, cut and bit-flipped, with capacities exact / +8 / -1 / 0, read in one call for both single values:
    every stream's result, src_consumed and content are the host reader's and the restated reader's for that stream alone,
    content_len is the content on success and after -9, nothing outside a stream's range is written, nothing at all in the
    range of a stream that fails.  Every -9 stream read again with dst_cap = content_len succeeds."""
    L, M = b200._native.lib(), _DevMem()
    rng = random.Random(2024)
    blobs = _cases(b200, port, rng, 30 if SIM else 400)
    full = [max(_host(L, b, BIG, False)[0], 0) for b in blobs]
    caps = [max(rng.choice((f, f, f + 8, f - 1, 0)), 0) for f in full]
    seen = {}
    for single in (False, True):
        res, used, content, dst, doff = _read_all(L, M, blobs, caps, single)
        _check(L, port, blobs, caps, single, res, used, content, dst, doff, seen)
        again = [k for k in range(len(blobs)) if res[k] == -9]
        assert again, single
        res2, _, _, _, _ = _read_all(L, M, [blobs[k] for k in again], [int(content[k]) for k in again], single)
        assert (res2 == content[again].astype(np.int64)).all(), (single, res2)
    assert {"ok", -1, -2, -3, -9} <= set(seen) and len([k for k in seen if k != "ok"]) >= (5 if SIM else 7), seen


def test_layout_freedom(b200, port):
    """sources at random byte phases with gaps, two streams over the same bytes, one stream inside another's range, and
    destinations in the reverse order of the sources"""
    L, M = b200._native.lib(), _DevMem()
    rng = random.Random(7)
    datas = [d for d in _datas(port) if len(d) <= (300000 if SIM else 1 << 22)]
    frames = [b200.compress_frame(d, 4 + k % 4, bool(k & 1), True, bool(k & 2)) for k, d in enumerate(datas)]
    offs, pos = [], rng.randrange(16)
    for f in frames:
        offs.append(pos)
        pos += len(f) + rng.randrange(1, 40)
    src = np.zeros(pos + 64, dtype=np.uint8)
    for o, f in zip(offs, frames):
        src[o:o + len(f)] = np.frombuffer(f, dtype=np.uint8)
    lens = [len(f) for f in frames]
    offs += [offs[3], offs[3], offs[1]]                                 # the same bytes twice more, and a prefix of a stream
    lens += [lens[3], lens[3], 9]
    want = datas + [datas[3], datas[3], None]
    caps = [len(d) if d is not None else 100 for d in want]
    doff, size = _dst_ranges(caps, order=list(reversed(range(len(caps)))))
    d_src, d_dst = M.up(src), M.full(size, GUARD)
    rc, res, used, content = _read(L, M, d_src, _u64(offs), _u64(lens), d_dst, doff, _u64(caps), False)
    out = M.down(d_dst)
    assert rc == 0
    for k, d in enumerate(want):
        if d is None:
            assert res[k] == -1 and used[k] == 0 and (out[doff[k]:doff[k] + 100] == GUARD).all(), res[k]
            continue
        assert res[k] == len(d) and used[k] == lens[k] and content[k] == len(d), (k, res[k])
        assert out[doff[k]:doff[k] + len(d)].tobytes() == d, k
    assert (out[:int(doff[-1])] == GUARD).all()


def test_room_and_content_len(b200, port):
    """dst_cap = content - 1: -9 with content_len right and nothing written; dst_cap = content_len then succeeds; dst_cap 0
    suits a stream whose content is empty (an empty frame, skippable frames only)"""
    L, M = b200._native.lib(), _DevMem()
    data = port.datagen(200000, 0.5, 0.0, 6).tobytes()
    good = b200.compress_frame(data, 4, True, True, True)
    flushed = _frame_of_pieces(port, [data[:60000], data[5:12], data[100:40000]], 4)
    two = good + SKIP + flushed
    empty = b200.compress_frame(b"", 5, True, False, True)
    blobs = [good, flushed, two, empty, SKIP, SKIP + empty]
    sizes = [len(data), 60000 + 7 + 39900, len(data) + 60000 + 7 + 39900, 0, 0, 0]
    for single in (False, True):
        want = [len(data), 99907, len(data) if single else sizes[2], 0, 0, 0]
        caps = [max(w - 1, 0) for w in want]
        res, used, content, dst, doff = _read_all(L, M, blobs, caps, single)
        assert res.tolist() == [-9, -9, -9, 0, 0, 0] and content.tolist() == want, (single, res, content)
        assert used.tolist()[3:] == [len(empty), len(SKIP), len(SKIP) + len(empty)]
        for k in range(3):
            assert (dst[doff[k]:doff[k] + caps[k] + 24] == GUARD).all(), k
        res, used, content, dst, doff = _read_all(L, M, blobs, [int(c) for c in content], single)
        assert res.tolist() == want and content.tolist() == want, (single, res)
        assert used.tolist()[:3] == [len(good), len(flushed), len(good) if single else len(two)]
        outs = [data, data[:60000] + data[5:12] + data[100:40000]]
        outs.append(outs[0] if single else outs[0] + outs[1])
        for k in range(3):
            assert dst[doff[k]:doff[k] + want[k]].tobytes() == outs[k] and (dst[doff[k] + want[k]:doff[k] + want[k] + 24] == GUARD).all()


def _write(L, M, datas, bs, flags, hc):
    """b200lz4f_compress_dev over the datas, sources at odd offsets -> (d_frames, frame_off, frame_len)"""
    src, offs, lens = _lay_out(datas, align=16, phase=7, gap=3)
    cap = sum(L.b200lz4f_compress_bound(int(n), bs) for n in lens)
    d_src, d_frames = M.up(src), M.full(cap + 64, 0)
    fo, fl = np.zeros(len(lens), dtype=np.uint64), np.zeros(len(lens), dtype=np.uint64)
    n = L.b200lz4f_compress_dev(M.ptr(d_src), offs.ctypes.data, lens.ctypes.data, len(lens), M.ptr(d_frames), cap,
                                fo.ctypes.data, fl.ctypes.data, bs, flags, hc, None)
    assert n == int(fl.sum()), (bs, flags, hc, n)
    return d_frames, fo, fl, lens


def test_round_trip_with_the_writer(b200, port):
    """b200lz4f_compress_dev's frame_off / frame_len fed straight back as src_off / src_len, bsCodes 4..7, flags 0..7, HC
    levels 1 and 9: every result is its source's length and the content is the source"""
    L, M = b200._native.lib(), _DevMem()
    data = port.datagen(100000 if SIM else 3000000, 0.5, 0.0, 4).tobytes()
    sizes = (70000, 0, 1, 5000) if SIM else (70000, 0, 1, 2000000, 65536, 0, 300001)
    datas = [data[k:k + n] for k, n in enumerate(sizes)]
    combos = [(bs, fl, hc) for bs in (4, 5, 6, 7) for fl in range(8) for hc in (1, 9)]
    if SIM:
        combos = [(4, 7, 1), (5, 0, 9), (7, 5, 1)]
    for bs, fl, hc in combos:
        d_frames, fo, fl_, lens = _write(L, M, datas, bs, fl, hc)
        doff, size = _dst_ranges(lens)
        d_dst = M.full(size, GUARD)
        for single in (False, True):
            rc, res, used, content = _read(L, M, d_frames, fo, fl_, d_dst, doff, lens, single)
            out = M.down(d_dst)
            assert rc == 0 and (res == lens.astype(np.int64)).all() and (used == fl_).all() and (content == lens).all(), (bs, fl, hc, res)
            for k, d in enumerate(datas):
                assert out[doff[k]:doff[k] + len(d)].tobytes() == d, (bs, fl, hc, k)


def test_errors_launch_nothing_and_write_nothing(b200, port):
    """NULL result or offsets, a destination range that overflows: B200LZ4_E_ARG before anything is launched, nothing written;
    no streams: 0"""
    L, M = b200._native.lib(), _DevMem()
    frames = [b200.compress_frame(port.datagen(100000, 0.5, 0.0, 6).tobytes(), 4, True, False, False), b"xyz"]
    src, offs, lens = _lay_out(frames)
    d_src, d_dst = M.up(src), M.full(200100, GUARD)
    doff, dcap = _u64([0, 100000]), _u64([100000, 3])
    before = L.b200lz4_launch_count()
    assert _read(L, M, d_src, offs, lens, d_dst, doff, dcap, False, result=False)[0] == E_ARG
    assert L.b200lz4f_decompress_streams_dev(M.ptr(d_src), None, lens.ctypes.data, 2, M.ptr(d_dst), doff.ctypes.data, dcap.ctypes.data,
                                             0, np.zeros(2, dtype=np.int64).ctypes.data, None, None, None) == E_ARG
    assert _read(L, M, d_src, offs, lens, d_dst, _u64([0, (1 << 64) - 2]), dcap, True)[0] == E_ARG
    assert L.b200lz4f_decompress_streams_dev(M.ptr(d_src), offs.ctypes.data, lens.ctypes.data, 2, None, doff.ctypes.data, dcap.ctypes.data,
                                             0, np.zeros(2, dtype=np.int64).ctypes.data, None, None, None) == E_ARG
    assert _read(L, M, d_src, offs[:0], lens[:0], d_dst, doff[:0], dcap[:0], False)[0] == 0
    assert L.b200lz4_launch_count() == before
    assert (M.down(d_dst) == GUARD).all()
    rc, res, used, content = _read(L, M, d_src, offs, lens, d_dst, doff, dcap, False)
    assert rc == 0 and res.tolist() == [100000, -1] and used.tolist() == [len(frames[0]), 0] and content.tolist() == [100000, 0]


def test_launches_do_not_depend_on_streams_frames_or_blocks(b200, port):
    """the same bytes as 1, 64 and 4096 one-frame streams (1, 4 and 16 on the emulator), and one stream of one 64-block frame
    against 64 one-block streams (16 on the emulator): the reader launches the same kernels"""
    L, M = b200._native.lib(), _DevMem()
    nb = 16 if SIM else 4096
    data = port.datagen(nb * 65536, 0.5, 0.0, 7).tobytes()
    counts = []
    splits = ((1, 4, 16) if SIM else (1, 64, 4096))
    for ns in splits:
        per = len(data) // ns
        d_frames, fo, fl, lens = _write(L, M, [data[k * per:(k + 1) * per] for k in range(ns)], 4, 7, 0)
        d_dst = M.full(len(data) + 64, GUARD)
        doff = _u64(np.arange(ns) * per)
        before = L.b200lz4_launch_count()
        rc, res, _, _ = _read(L, M, d_frames, fo, fl, d_dst, doff, lens, False)
        counts.append(L.b200lz4_launch_count() - before)
        assert rc == 0 and (res == per).all() and M.down(d_dst)[:len(data)].tobytes() == data, ns
    assert len(set(counts)) == 1, counts
    m = 16 if SIM else 64
    one = _frame_of_pieces(port, [data[k * 65536:(k + 1) * 65536] for k in range(m)], 4, block_checksum=True)
    many = [_frame_of_pieces(port, [data[k * 65536:(k + 1) * 65536]], 4, block_checksum=True) for k in range(m)]
    counts = []
    for blobs in ([one], many):
        src, offs, lens = _lay_out(blobs)
        caps = _u64([m * 65536] if len(blobs) == 1 else [65536] * m)
        doff = _u64(np.cumsum(caps) - caps)
        d_src, d_dst = M.up(src), M.full(m * 65536 + 64, GUARD)
        before = L.b200lz4_launch_count()
        rc, res, _, _ = _read(L, M, d_src, offs, lens, d_dst, doff, caps, False)
        counts.append(L.b200lz4_launch_count() - before)
        assert rc == 0 and (res == caps.astype(np.int64)).all() and M.down(d_dst)[:m * 65536].tobytes() == data[:m * 65536]
    assert counts[0] == counts[1], counts


@pytest.mark.skipif(not SIM, reason="the counting emulator build counts the library's host<->device copies")
def test_no_payload_crosses_to_the_host(b200, port):
    """two calls with the same streams and frames whose payloads differ 16x in size: the reader copies the same bytes between
    host and device for both, far fewer than one stream holds (on the counting emulator library, tests/simt/copy_count.h,
    which test_frame_streams_sim.py builds)"""
    L, M = b200._native.lib(), _DevMem()
    if not hasattr(L, "b200lz4_sim_copied_bytes"):
        pytest.skip("this emulator library does not count copies: tests/simt/copy_count.h")
    L.b200lz4_sim_copied_bytes.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
    h2d, d2h = ctypes.c_ulonglong(0), ctypes.c_ulonglong(0)
    rng = random.Random(8)
    counts = []
    for size in (4096, 65536):
        frame = lambda: _frame_of_pieces(port, [rng.randbytes(size) for _ in range(4)], 4, block_checksum=True, stored=set(range(4)))
        blobs = [frame(), SKIP + frame() + SKIP, frame() + frame(), frame()[:-3]]
        caps = [4 * size, 4 * size, 8 * size, 4 * size]
        src, offs, lens = _lay_out(blobs)
        doff = _u64(np.cumsum(caps) - caps)
        d_src, d_dst = M.up(src), M.full(sum(caps) + 64, 0)
        L.b200lz4_sim_copied_bytes(ctypes.byref(h2d), ctypes.byref(d2h))
        a = (h2d.value, d2h.value)
        rc, res, _, _ = _read(L, M, d_src, offs, lens, d_dst, doff, _u64(caps), False)
        L.b200lz4_sim_copied_bytes(ctypes.byref(h2d), ctypes.byref(d2h))
        counts.append((h2d.value - a[0], d2h.value - a[1]))
        assert rc == 0 and res.tolist() == caps[:3] + [-1], res
    assert counts[0] == counts[1], counts
    assert 0 < counts[0][0] and 0 < counts[0][1] and sum(counts[0]) < 4 * 4096, counts


@pytest.mark.skipif(SIM, reason="torch streams: GPU only")
def test_ordered_after_a_side_stream(b200, port):
    """the streams are written by a torch op on a side stream and the call is made on that stream without a synchronise: it
    reads the new bytes"""
    import torch
    old_data, new_data = port.datagen(3 << 20, 0.5, 0.0, 1).tobytes(), port.datagen(3 << 20, 0.5, 0.0, 2).tobytes()
    pieces = lambda d: [d[:1 << 20], d[1 << 20:]]
    old = [b200.compress_frame(p, 4, True, True, False) for p in pieces(old_data)]
    new = [b200.compress_frame(p, 4, True, True, False) for p in pieces(new_data)]
    n = max(len(old[0]) + len(old[1]), len(new[0]) + len(new[1]))
    pad = lambda fs: np.frombuffer(b"".join(fs) + bytes(n - len(b"".join(fs))), dtype=np.uint8)
    d_src, d_new = torch.from_numpy(pad(old).copy()).cuda(), torch.from_numpy(pad(new).copy()).cuda()
    out = torch.full((len(new_data),), GUARD, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.cuda._sleep(20_000_000)                                   # the copy lands well after the call is made
        d_src.copy_(d_new)
        res, used, content = b200.decompress_frame_streams_dev(d_src, [0, len(new[0])], [len(new[0]), len(new[1])], out,
                                                               [0, 1 << 20], [1 << 20, 2 << 20])
    torch.cuda.synchronize()
    assert res.tolist() == [1 << 20, 2 << 20] and out.cpu().numpy().tobytes() == new_data


@pytest.mark.skipif(SIM, reason="torch tensors: GPU only")
def test_python_wrapper(b200, port):
    import torch
    data = port.datagen(300003, 0.5, 0.0, 9)
    datas = [data[:300000].tobytes(), b"", data[300000:].tobytes()]
    src = torch.from_numpy(data.copy()).cuda()
    frames, fo, fl = b200.compress_frames_dev(src, [0, 0, 300000], [300000, 0, 3], 5, True, True, True)
    frames = torch.cat([frames, frames])                              # the frames twice: a second copy of every stream
    out = torch.full((400000,), GUARD, dtype=torch.uint8, device="cuda")
    res, used, content = b200.decompress_frame_streams_dev(frames, list(fo) + [int(fo[0]) + len(frames) // 2],
                                                           list(fl) + [int(fl[0])], out, [0, 300000, 300100, 300200],
                                                           [300000, 10, 2, 99000])
    assert res.dtype == np.int64 and used.dtype == np.uint64 and content.dtype == np.uint64
    assert res.tolist() == [300000, 0, -9, -9] and content.tolist() == [300000, 0, 3, 300000]
    assert used.tolist() == [int(fl[0]), int(fl[1]), 0, 0]
    host = out.cpu().numpy()
    assert host[:300000].tobytes() == datas[0] and (host[300000:] == GUARD).all()
    res, _, _ = b200.decompress_frame_streams_dev(frames, fo, fl, out, [0, 300000, 300100], [300000, 0, 3], read_single_frame=True)
    assert res.tolist() == [300000, 0, 3] and out[300100:300103].cpu().numpy().tobytes() == datas[2]
    with pytest.raises(ValueError):
        b200.decompress_frame_streams_dev(frames.cpu(), fo, fl, out, [0, 0, 0], [1, 1, 1])
    with pytest.raises(ValueError):
        b200.decompress_frame_streams_dev(frames, fo, fl, out.cpu(), [0, 0, 0], [1, 1, 1])
    with pytest.raises(ValueError):
        b200.decompress_frame_streams_dev(frames, fo, fl, out, [0, 0], [1, 1])
    with pytest.raises(ValueError):
        b200.decompress_frame_streams_dev(frames, fo, fl, out, [0, 0, 0], [1, 1, 400001])
    with pytest.raises(ValueError):
        b200.decompress_frame_streams_dev(frames, [0, 0, len(frames)], fl, out, [0, 0, 0], [1, 1, 1])
