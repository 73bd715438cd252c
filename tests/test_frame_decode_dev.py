"""b200lz4f_index_create_dev / b200lz4f_decompress_dev: the LZ4 Frame reader for containers in device memory.  The device
index must be the host indexer's (b200lz4f_index_create[_single]) on the same bytes, whatever hints are given, and
decompress_dev must return what decompress_host returns.  Runs on the H100, and on the CPU emulator build of the library
(B200LZ4_TEST_SO=.../libb200lz4_sim.so), where the sizes shrink and torch is not used."""
import ctypes
import os
import random

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SIM = "sim" in os.environ.get("B200LZ4_TEST_SO", "")
E_ARG = -2147483645
SKIP = bytes([0x5A, 0x2A, 0x4D, 0x18, 3, 0, 0, 0, 9, 9, 9])          # a skippable frame of 3 bytes


class _DevMem:
    """device buffers for the C ABI: torch CUDA tensors on a GPU box, numpy arrays under the emulator build (its "device
    memory" is the host heap)"""

    def __init__(self):
        if not SIM:
            import torch
            self.torch = torch

    def up(self, arr):
        arr = np.ascontiguousarray(arr)
        if SIM:
            return arr.copy()
        return self.torch.from_numpy(arr.view(np.uint8).reshape(-1).copy()).cuda()

    def full(self, nbytes, value):
        return self.up(np.full(max(nbytes, 16), value, dtype=np.uint8))

    def ptr(self, buf):
        return buf.ctypes.data if SIM else buf.data_ptr()

    def down(self, buf):
        if not SIM:
            self.torch.cuda.synchronize()
            buf = buf.cpu().numpy()
        return buf.view(np.uint8).reshape(-1)


def _src(M, blob):
    """the container in device memory, with slack behind it (the decoders read whole aligned words)"""
    return M.up(np.concatenate([np.frombuffer(bytes(blob), dtype=np.uint8), np.zeros(64, dtype=np.uint8)]))


def _hints(h):
    return None if h is None else np.ascontiguousarray(np.asarray(h, dtype=np.uint64).reshape(-1))


def _index(L, M, blob, single, hints=None, dev=True, d_src=None):
    """(handle, err, slot_bytes, src_consumed) from the host or the device indexer"""
    slot, err, used = ctypes.c_uint64(0), ctypes.c_int(0), ctypes.c_size_t(0)
    if dev:
        h = _hints(hints)
        d_src = _src(M, blob) if d_src is None else d_src
        ix = L.b200lz4f_index_create_dev(M.ptr(d_src), len(blob), int(single), h.ctypes.data if h is not None and len(h) else None,
                                         0 if h is None else len(h), ctypes.byref(slot), ctypes.byref(used), ctypes.byref(err), None)
    else:
        src = np.frombuffer(bytes(blob), dtype=np.uint8) if blob else np.zeros(1, dtype=np.uint8)
        if single:
            ix = L.b200lz4f_index_create_single(src.ctypes.data, len(blob), ctypes.byref(slot), ctypes.byref(used), ctypes.byref(err))
        else:
            ix = L.b200lz4f_index_create(src.ctypes.data, len(blob), ctypes.byref(slot), ctypes.byref(err))
    return ix, err.value, slot.value, used.value


def _facts(L, M, blob, single, hints=None, dev=True):
    """everything an index says and what decode_dev makes of it"""
    ix, err, slot, used = _index(L, M, blob, single, hints, dev)
    if not ix:
        return (err, used if single else None)
    nf, nb = L.b200lz4f_index_frames(ix), L.b200lz4f_index_blocks(ix)
    offs = np.zeros(max(nb, 1), dtype=np.uint64)
    L.b200lz4f_index_block_offsets(ix, offs.ctypes.data)
    d_src, d_slots = _src(M, blob), M.full(slot + 64, 0)
    fo, fl, bl = np.zeros(max(nf, 1), dtype=np.uint64), np.zeros(max(nf, 1), dtype=np.uint64), np.zeros(max(nb, 1), dtype=np.int32)
    rc = L.b200lz4f_decode_dev(ix, M.ptr(d_src), M.ptr(d_slots), fo.ctypes.data, fl.ctypes.data, bl.ctypes.data, None)
    slots = M.down(d_slots).tobytes()
    L.b200lz4f_index_free(ix)
    return (err, used if single else None, slot, nf, nb, offs[:nb].tolist(), rc, fo[:nf].tolist(), fl[:nf].tolist(),
            bl[:nb].tolist() if rc >= 0 or rc == -11 else None, slots)


def _same_index(L, M, blob, single=False, hints=None):
    want = _facts(L, M, blob, single, dev=False)
    got = _facts(L, M, blob, single, hints, dev=True)
    assert got == want, (len(blob), single, hints, got[:10], want[:10])
    return got


def _decompress_dev(L, M, blob, cap, single=False, hints=None, d_src=None):
    """-> (rc, d_dst contents (filled with 0xAA before), src_consumed)"""
    d_src = _src(M, blob) if d_src is None else d_src
    d_dst = M.full(cap + 64, 0xAA)
    h = _hints(hints)
    used = ctypes.c_size_t(0)
    rc = L.b200lz4f_decompress_dev(M.ptr(d_src), len(blob), M.ptr(d_dst), cap, int(single), h.ctypes.data if h is not None and len(h) else None,
                                   0 if h is None else len(h), ctypes.byref(used), None)
    return rc, M.down(d_dst), used.value


def _frame_of_pieces(port, pieces, bs_code, content_checksum=True, block_checksum=False, stored=()):
    """an LZ4 frame whose blocks are exactly `pieces` (what LZ4FrameOutputStream writes when flush() is called between
    writes): short blocks anywhere, stored when they do not shrink or when asked"""
    hdr = bytes([0x60 | (0x10 if block_checksum else 0) | (0x04 if content_checksum else 0), bs_code << 4])
    out = bytearray(b"\x04\x22\x4d\x18" + hdr + bytes([(port.xxh32(hdr, 0) >> 8) & 0xFF]))
    for i, piece in enumerate(pieces):
        c = port.compress(piece)
        raw = i in stored or len(c) >= len(piece)
        payload = piece if raw else c
        out += (len(payload) | (0x80000000 if raw else 0)).to_bytes(4, "little") + payload
        if block_checksum:
            out += port.xxh32(payload, 0).to_bytes(4, "little")
    out += (0).to_bytes(4, "little")
    if content_checksum:
        out += port.xxh32(b"".join(pieces), 0).to_bytes(4, "little")
    return bytes(out)


def _concat(frames):
    """the container and where each frame starts"""
    offs, pos = [], 0
    for f in frames:
        offs.append(pos)
        pos += len(f)
    return b"".join(frames), offs


def _datas(port):
    rdg = port.datagen(1 << 20, 0.5, 0.0, 3).tobytes()
    sizes = (0, 1, 100, 65536, 65537, 300000) if SIM else (0, 1, 100, 65535, 65536, 65537, 300000, 3 * (1 << 20) + 5)
    datas = [(rdg * 4)[:n] for n in sizes]
    datas.append(random.Random(11).randbytes(100000))                      # does not shrink: stored blocks
    return datas


def test_index_parity_on_writer_output(b200, port):
    """frames as the writers write them, every bsCode 4..7 and flags 0..7 (a subset on the emulator): the same index and
    decode with no hints, with the frame starts as hints, and read single"""
    L, M = b200._native.lib(), _DevMem()
    datas = _datas(port)
    combos = [(bs, fl) for bs in (4, 5, 6, 7) for fl in range(8)]
    if SIM:
        combos = [(4, 0), (4, 7), (5, 3), (7, 6)]
    for bs, fl in combos:
        blob, offs = _concat([b200.compress_frame(d, bs, bool(fl & 1), bool(fl & 2), bool(fl & 4)) for d in datas])
        got = _same_index(L, M, blob)
        assert got[0] == 0 and got[6] == sum(map(len, datas)), (bs, fl, got[:1], got[6])
        assert _same_index(L, M, blob, hints=offs) == got
        _same_index(L, M, blob, single=True, hints=offs)


def test_index_parity_on_flushed_frames_and_skippable_frames(b200, port):
    """short blocks mid-frame (-11 from decode_dev), skippable frames before, between and after frames, a container of
    skippable frames only, the empty container, and `single` on concatenations"""
    L, M = b200._native.lib(), _DevMem()
    rng = random.Random(5)
    base = port.datagen(1 << 19, 0.5, 0.0, 9).tobytes()
    flushed = []
    for trial in range(3 if SIM else 8):
        bs_code = rng.choice((4, 5, 6, 7))
        sizes = [rng.choice((1, 5, 16, 17, 100, 4097, 65535, 65536)) for _ in range(rng.randrange(1, 12 if SIM else 30))]
        pieces = [(base * 2)[o:o + n] for o, n in ((rng.randrange(0, len(base)), n) for n in sizes)]
        flushed.append(_frame_of_pieces(port, pieces, bs_code, content_checksum=trial % 3 != 2, block_checksum=bool(trial & 1),
                                        stored={i for i in range(len(pieces)) if rng.random() < 0.15}))
    plain = b200.compress_frame(base[:150000], 4, True, True, False)
    for f in flushed:
        assert _same_index(L, M, f)[6] == -11
    cases = [
        SKIP + flushed[0] + SKIP + plain + SKIP + SKIP + flushed[1] + SKIP,
        SKIP, SKIP * 3, b"",
        plain + flushed[2] + plain,
        SKIP + plain + plain + b"\x00garbage that is not a frame",
    ]
    for blob in cases:
        for single in (False, True):
            _same_index(L, M, blob, single)
            _same_index(L, M, blob, single, hints=[len(SKIP)] if len(blob) > len(SKIP) else None)


def _faulty(rng, port, base):
    """the generator of the stream-order test: 1-3 frames of either writer, then 1-3 cuts and bit flips"""
    frames = []
    for _ in range(rng.randrange(1, 4)):
        pieces = [base[o:o + n] for o, n in ((rng.randrange(0, 100000), rng.choice((1, 40, 700, 5000, 65536))) for _ in range(rng.randrange(0, 5)))]
        if rng.random() < 0.5:
            frames.append(port.frame_compress(b"".join(pieces), rng.choice((4, 5)), rng.randrange(8)))
        else:
            frames.append(_frame_of_pieces(port, pieces, rng.choice((4, 5)), content_checksum=rng.random() < 0.7, block_checksum=rng.random() < 0.5,
                                           stored={i for i in range(len(pieces)) if rng.random() < 0.2}))
    blob = bytearray(b"".join(frames))
    for _ in range(rng.randrange(1, 4)):
        kind = rng.randrange(4)
        if kind == 0 and len(blob) > 8:
            del blob[rng.randrange(len(blob) - 8, len(blob)):]
        elif kind == 1 and len(blob) > 1:
            del blob[rng.randrange(1, len(blob)):]
        elif blob:
            i = rng.randrange(len(blob)); blob[i] ^= 1 << rng.randrange(8)
    return bytes(blob)


def test_errors_come_in_stream_order(b200, port):
    """random faults: decompress_dev returns the restated LZ4FrameInputStream's code, which is decompress_host's, and on
    success the same bytes; d_dst is not written at all on an error, and not past the total on success"""
    L, M = b200._native.lib(), _DevMem()
    rng = random.Random(2024)
    base = port.datagen(1 << 18, 0.5, 0.0, 21).tobytes()
    seen = {}
    cap = 1 << 20
    for trial in range(60 if SIM else 400):
        blob = _faulty(rng, port, base)
        want, out = port.frame_decompress(blob, cap)
        try:
            host = len(b200.decompress_frames(blob, cap))
        except b200.LZ4FrameError as e:
            host = e.code
        assert host == want, (trial, host, want)
        rc, dst, _ = _decompress_dev(L, M, blob, cap)
        assert rc == want, (trial, rc, want)
        if want >= 0:
            assert dst[:rc].tobytes() == out and (dst[rc:] == 0xAA).all(), trial
        else:
            assert (dst == 0xAA).all(), trial
        seen[want if want < 0 else "ok"] = seen.get(want if want < 0 else "ok", 0) + 1
    assert len([k for k in seen if k != "ok"]) >= (4 if SIM else 6), seen


def test_hints_never_change_the_result(b200, port):
    """correct hints, hints inside payloads, a hint at 0, on a skippable frame and behind the last frame: the index of no
    hints.  Unsorted hints or hints at or past srcSize: B200LZ4_E_ARG before anything is launched."""
    L, M = b200._native.lib(), _DevMem()
    rng = random.Random(3)
    datas = _datas(port)
    blob, offs = _concat([b200.compress_frame(d, 4, True, True, bool(k & 1)) for k, d in enumerate(datas)])
    blob += SKIP
    skip_at = len(blob) - len(SKIP)
    blob += b200.compress_frame(datas[3], 5, True, False, False)
    last = offs[-1]
    want = _same_index(L, M, blob)
    inside = sorted(rng.randrange(1, len(blob)) for _ in range(6))
    for hints in (offs, inside, [0], [0, 0] + offs[1:3], [skip_at], [last + 1, len(blob) - 1], sorted(offs + inside + [skip_at])):
        assert _same_index(L, M, blob, hints=hints) == want, hints
        rc, dst, _ = _decompress_dev(L, M, blob, sum(map(len, datas)) + len(datas[3]), hints=hints)
        assert rc == want[6] and dst[:rc].tobytes() == b"".join(datas) + datas[3], hints
    d_src = _src(M, blob)
    before = L.b200lz4_launch_count()
    for bad in ([5, 4], [len(blob)], [0, len(blob) + 7]):
        ix, err, _, _ = _index(L, M, blob, False, bad, d_src=d_src)
        assert not ix and err == E_ARG, bad
        assert _decompress_dev(L, M, blob, 1 << 20, hints=bad, d_src=d_src)[0] == E_ARG, bad
    assert L.b200lz4_launch_count() == before


def test_device_round_trip_with_the_writer(b200, port):
    """b200lz4f_compress_dev -> b200lz4f_decompress_dev with frame_off as hints gives back the sources: bsCodes 4..7, HC
    level 9, empty frames, sources at unaligned offsets"""
    L, M = b200._native.lib(), _DevMem()
    data = port.datagen(400000 if SIM else 3000000, 0.5, 0.0, 4).tobytes()
    datas = [data[:n] for n in ((70000, 0, 1, 200000, 65536) if SIM else (70000, 0, 1, 2000000, 65536, 0))]
    for phase, bs, hc in ((0, 4, 0), (3, 5, 0), (1, 6, 9), (7, 7, 0)):
        offs, pos = [], phase
        for d in datas:
            offs.append(pos)
            pos += len(d) + 13
        src = np.zeros(pos + 64, dtype=np.uint8)
        for o, d in zip(offs, datas):
            src[o:o + len(d)] = np.frombuffer(d, dtype=np.uint8)
        offs, lens = np.asarray(offs, dtype=np.uint64), np.asarray([len(d) for d in datas], dtype=np.uint64)
        cap = sum(L.b200lz4f_compress_bound(int(n), bs) for n in lens)
        d_src, d_frames = M.up(src), M.full(cap + 64, 0)
        fo, fl = np.zeros(len(lens), dtype=np.uint64), np.zeros(len(lens), dtype=np.uint64)
        n = L.b200lz4f_compress_dev(M.ptr(d_src), offs.ctypes.data, lens.ctypes.data, len(lens), M.ptr(d_frames), cap,
                                    fo.ctypes.data, fl.ctypes.data, bs, 7, hc, None)
        assert n == int(fl.sum()), (phase, bs, hc)
        h = np.ascontiguousarray(fo)
        d_dst = M.full(len(data) + 64, 0xAA)
        used = ctypes.c_size_t(0)
        rc = L.b200lz4f_decompress_dev(M.ptr(d_frames), n, M.ptr(d_dst), len(data), 0, h.ctypes.data, len(h), ctypes.byref(used), None)
        out = M.down(d_dst)
        assert rc == sum(map(len, datas)) and out[:rc].tobytes() == b"".join(datas) and (out[rc:] == 0xAA).all(), (phase, bs, hc, rc)


def test_nothing_written_where_it_should_not_be(b200, port):
    """0xAA in d_dst: untouched past the total after success, and entirely after every error code, -9 included"""
    L, M = b200._native.lib(), _DevMem()
    data = port.datagen(200000, 0.5, 0.0, 6).tobytes()
    good = b200.compress_frame(data, 4, True, True, True)
    flushed = _frame_of_pieces(port, [data[:60000], data[5:12], data[100:40000]], 4)
    for blob, n in ((good, len(data)), (flushed, 60000 + 7 + 39900)):
        rc, dst, _ = _decompress_dev(L, M, blob, n)
        assert rc == n and (dst[n:] == 0xAA).all()
        rc, dst, _ = _decompress_dev(L, M, blob, n - 1)
        assert rc == -9 and (dst == 0xAA).all()
    hdr_bad = bytearray(good); hdr_bad[6] ^= 1                                   # header checksum byte
    blk_bad = bytearray(good); blk_bad[15 + 4 + 100] ^= 0x10                    # inside the first block's payload
    for blob, code in ((good[:-3], -1), (b"abcd" + good, -2), (bytes(hdr_bad), -3), (good[:4] + bytes([good[4] ^ 0x80]) + good[5:], -10),
                       (bytes(blk_bad), None)):
        rc, dst, _ = _decompress_dev(L, M, blob, len(data))
        assert rc < 0 and (code is None or rc == code), (code, rc)
        assert (dst == 0xAA).all(), code


@pytest.mark.skipif(not SIM, reason="the counting emulator build counts the library's host<->device copies")
def test_no_payload_crosses_to_the_host(b200, port):
    """two containers of the same frame and block structure whose payloads differ 16x in size: the device indexer and
    decompress_dev copy the same bytes between host and device for both, far fewer than the container holds (on the
    counting emulator library, tests/simt/copy_count.h, which test_frame_decode_sim.py builds)"""
    L, M = b200._native.lib(), _DevMem()
    if not hasattr(L, "b200lz4_sim_copied_bytes"):
        pytest.skip("this emulator library does not count copies: tests/simt/copy_count.h")
    rng = random.Random(8)
    small = _frame_of_pieces(port, [rng.randbytes(4096) for _ in range(8)], 4, stored=set(range(8)))
    large = _frame_of_pieces(port, [rng.randbytes(65536) for _ in range(8)], 4, stored=set(range(8)))
    both = [(c + SKIP + c, h) for c, h in ((small, None), (large, None), (small, [len(small)]), (large, [len(large)]))]
    h2d, d2h = ctypes.c_ulonglong(0), ctypes.c_ulonglong(0)

    def copied(fn):
        L.b200lz4_sim_copied_bytes(ctypes.byref(h2d), ctypes.byref(d2h))
        a = (h2d.value, d2h.value)
        fn()
        L.b200lz4_sim_copied_bytes(ctypes.byref(h2d), ctypes.byref(d2h))
        return h2d.value - a[0], d2h.value - a[1]

    L.b200lz4_sim_copied_bytes.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
    for fn in ("index", "decompress"):
        counts = []
        for blob, hints in both:
            d_src = _src(M, blob)
            if fn == "index":
                def run():
                    ix, err, _, _ = _index(L, M, blob, False, hints, d_src=d_src)
                    assert ix and err == 0
                    L.b200lz4f_index_free(ix)
            else:
                def run():
                    assert _decompress_dev(L, M, blob, 16 * 65536 + 64, hints=hints, d_src=d_src)[0] in (16 * 4096, 16 * 65536)
            counts.append(copied(run))
        assert counts[0] == counts[1] and counts[2] == counts[3], (fn, counts)
        assert all(0 < c[0] and 0 < c[1] and sum(c) < len(small) for c in counts), (fn, counts)


def test_index_launches_do_not_depend_on_frames(b200, port):
    """one frame of 64 blocks and 64 one-block frames: the device indexer launches the same kernels, with and without hints"""
    L, M = b200._native.lib(), _DevMem()
    n = 16 if SIM else 64
    data = port.datagen(n * 65536, 0.5, 0.0, 7).tobytes()
    one = [b200.compress_frame(data, 4, True, False, False)]
    many = [b200.compress_frame(data[k * 65536:(k + 1) * 65536], 4, True, False, False) for k in range(n)]
    for with_hints in (False, True):
        counts = []
        for frames in (one, many):
            blob, offs = _concat(frames)
            d_src = _src(M, blob)
            before = L.b200lz4_launch_count()
            ix, err, _, _ = _index(L, M, blob, False, offs if with_hints else None, d_src=d_src)
            counts.append(L.b200lz4_launch_count() - before)
            assert ix and err == 0 and L.b200lz4f_index_blocks(ix) == n
            L.b200lz4f_index_free(ix)
        assert counts[0] == counts[1], (with_hints, counts)


def test_freeing_an_index_leaves_the_current_device(b200, port, monkeypatch):
    """an index decoded on device 1 and freed after the thread went back to device 0: the current device stays 0, because
    freeing an index makes no CUDA call.  Two pretend devices on the emulator, two GPUs on a GPU box."""
    L, M = b200._native.lib(), _DevMem()
    if SIM:
        if not hasattr(L, "b200lz4_sim_current_device"):
            pytest.skip("this emulator library has no current-device accessor: tests/simt/copy_count.cpp")
        monkeypatch.setenv("SIMT_DEVICES", "2")
        current = L.b200lz4_sim_current_device
    else:
        import torch
        if torch.cuda.device_count() < 2:
            pytest.skip("needs two GPUs")
        current = torch.cuda.current_device
    data = port.datagen(100000, 0.5, 0.0, 12).tobytes()
    blob = b200.compress_frame(data, 4, True, True, False)
    ix, err, slot, _ = _index(L, M, blob, False, dev=False)
    assert ix and err == 0
    try:
        assert L.b200lz4_set_device(1) == 0
        d_src, d_slots = _src(M, blob), M.full(slot + 64, 0)              # memory of device 1, the current one now
        assert L.b200lz4f_decode_dev(ix, M.ptr(d_src), M.ptr(d_slots), None, None, None, None) == len(data)
        assert M.down(d_slots)[:len(data)].tobytes() == data
        assert L.b200lz4_set_device(0) == 0
        L.b200lz4f_index_free(ix)
        assert current() == 0
    finally:
        L.b200lz4_set_device(0)


def test_one_index_decoded_by_several_threads(b200, port):
    """four threads decode one index at once, each into its own slots and on its own stream, many times over: every decode
    gives what one thread alone gets (decode_dev only reads the index)"""
    import threading
    L, M = b200._native.lib(), _DevMem()
    base = port.datagen(1 << 19, 0.5, 0.0, 13).tobytes()
    frames = [b200.compress_frame(base[:n], 4, True, True, True) for n in ((70000, 1, 5000) if SIM else (3000000, 1, 70000))]
    frames.append(_frame_of_pieces(port, [base[:5000], base[7:100], base[200:60000]], 4, block_checksum=True, stored={1}))
    blob = SKIP.join(frames)
    ix, err, slot, _ = _index(L, M, blob, False, dev=False)
    assert ix and err == 0
    nf, nb = L.b200lz4f_index_frames(ix), L.b200lz4f_index_blocks(ix)
    d_src = _src(M, blob)
    if not SIM:
        import torch
        torch.cuda.synchronize()

    def decode(stream=None):
        d_slots = M.full(slot + 64, 0)
        if stream is not None:
            stream.wait_stream(torch.cuda.current_stream())                  # the slots are filled on this thread's stream
        fo, fl, bl = np.zeros(nf, dtype=np.uint64), np.zeros(nf, dtype=np.uint64), np.zeros(nb, dtype=np.int32)
        rc = L.b200lz4f_decode_dev(ix, M.ptr(d_src), M.ptr(d_slots), fo.ctypes.data, fl.ctypes.data, bl.ctypes.data,
                                   None if stream is None else stream.cuda_stream)
        return rc, fo.tolist(), fl.tolist(), bl.tolist(), M.down(d_slots).tobytes()

    want = decode()
    assert want[0] == -11, want[0]
    got = [[] for _ in range(4)]

    def worker(k):
        stream = None if SIM else torch.cuda.Stream()
        for _ in range(3 if SIM else 30):
            got[k].append(decode(stream))

    threads = [threading.Thread(target=worker, args=(k,)) for k in range(4)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    L.b200lz4f_index_free(ix)
    assert all(len(g) == (3 if SIM else 30) and all(r == want for r in g) for g in got), [[r[0] for r in g] for g in got]


_FAILED_PINNED = r"""
import ctypes, os, sys
import numpy as np
lib = ctypes.CDLL(sys.argv[1])
vp = ctypes.c_void_p
lib.b200lz4f_index_create.restype, lib.b200lz4f_index_create.argtypes = vp, [vp, ctypes.c_size_t, vp, vp]
lib.b200lz4f_decode_dev.restype, lib.b200lz4f_decode_dev.argtypes = ctypes.c_int64, [vp] * 7
lib.b200lz4f_index_free.argtypes = [vp]
lib.b200lz4_last_error.restype = ctypes.c_char_p
blob, data = (np.fromfile(f, dtype=np.uint8) for f in sys.argv[2:4])
slot, err = ctypes.c_uint64(0), ctypes.c_int(0)
ix = lib.b200lz4f_index_create(blob.ctypes.data, len(blob), ctypes.byref(slot), ctypes.byref(err))
assert ix and err.value == 0, err.value
d_src = np.concatenate([blob, np.zeros(64, dtype=np.uint8)])
def decode():
    d_slots, fo, fl = np.zeros(slot.value + 64, dtype=np.uint8), np.zeros(1, dtype=np.uint64), np.zeros(1, dtype=np.uint64)
    rc = lib.b200lz4f_decode_dev(ix, d_src.ctypes.data, d_slots.ctypes.data, fo.ctypes.data, fl.ctypes.data, None, None)
    return rc, d_slots[int(fo[0]):int(fo[0] + fl[0])]
os.environ["SIMT_FAIL_HOST_ALLOC"] = "1"
rc, _ = decode()                            # the thread's first decode: its pinned scratch cannot be allocated
del os.environ["SIMT_FAIL_HOST_ALLOC"]
assert rc == -2147483646 and b"cudaHostAlloc" in lib.b200lz4_last_error(), (rc, lib.b200lz4_last_error())
rc, out = decode()
assert rc == len(data) and out.tobytes() == data.tobytes(), rc
lib.b200lz4f_index_free(ix)
print("ok")
"""


@pytest.mark.skipif(not SIM, reason="the emulator build can make pinned allocations fail (SIMT_FAIL_HOST_ALLOC)")
def test_failed_pinned_allocation_leaves_the_index_usable(b200, port, tmp_path):
    """decode_dev whose pinned scratch cannot be allocated returns B200LZ4_E_CUDA and names cudaHostAlloc; the same index then
    decodes correctly.  In a fresh process, whose thread has no pinned scratch yet."""
    import subprocess
    import sys
    data = port.datagen(200000, 0.5, 0.0, 14).tobytes()
    (tmp_path / "blob").write_bytes(b200.compress_frame(data, 4, True, True, False))
    (tmp_path / "data").write_bytes(data)
    r = subprocess.run([sys.executable, "-c", _FAILED_PINNED, os.environ["B200LZ4_TEST_SO"], str(tmp_path / "blob"), str(tmp_path / "data")],
                       capture_output=True, text=True)
    assert r.returncode == 0 and r.stdout.strip() == "ok", (r.returncode, r.stdout[-2000:] + r.stderr[-2000:])


@pytest.mark.skipif(SIM, reason="torch streams: GPU only")
def test_ordered_after_the_stream(b200, port):
    """the container is written by a torch op on a side stream and decompress_frames_dev is called on that stream without a
    synchronise: it reads the new bytes"""
    import torch
    old_data, new_data = port.datagen(3 << 20, 0.5, 0.0, 1).tobytes(), port.datagen(3 << 20, 0.5, 0.0, 2).tobytes()
    old, new = b200.compress_frame(old_data, 4, True, True, False), b200.compress_frame(new_data, 4, True, True, False)
    n = max(len(old), len(new))
    pad = lambda f: np.frombuffer(f + bytes(n - len(f)), dtype=np.uint8)
    d_src, d_new = torch.from_numpy(pad(old).copy()).cuda(), torch.from_numpy(pad(new).copy()).cuda()
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.cuda._sleep(20_000_000)                          # the copy lands well after the call is made
        d_src.copy_(d_new)
        got = b200.decompress_frames_dev(d_src[:len(new)], len(new_data))
    torch.cuda.synchronize()
    assert got.cpu().numpy().tobytes() == new_data


@pytest.mark.skipif(SIM, reason="torch tensors: GPU only")
def test_python_wrapper(b200, port):
    import torch
    datas = [port.datagen(300000, 0.5, 0.0, 9).tobytes(), b"", b"abc"]
    blob, offs = _concat([b200.compress_frame(d, 5, False, True, True) for d in datas])
    src = torch.from_numpy(np.frombuffer(blob, dtype=np.uint8).copy()).cuda()
    want = b200.decompress_frames(src.cpu().numpy(), 400000)
    got = b200.decompress_frames_dev(src, 400000)
    assert got.is_cuda and got.cpu().numpy().tobytes() == want == b"".join(datas)
    assert b200.decompress_frames_dev(src, 400000, frame_hints=offs).cpu().numpy().tobytes() == want
    assert b200.decompress_frames_dev(src, 400000, read_single_frame=True).cpu().numpy().tobytes() == datas[0]
    out = torch.full((400100,), 0xAA, dtype=torch.uint8, device="cuda")
    got2 = b200.decompress_frames_dev(src, 400000, out=out)
    assert got2.data_ptr() == out.data_ptr() and got2.cpu().numpy().tobytes() == want and (out[len(want):] == 0xAA).all()
    for bad, code in ((src[:-2], -1), (src[4:], -2)):
        with pytest.raises(b200.LZ4FrameError) as e:
            b200.decompress_frames_dev(bad.contiguous(), 400000)
        with pytest.raises(b200.LZ4FrameError) as e2:
            b200.decompress_frames(bad.cpu().numpy(), 400000)
        assert e.value.code == e2.value.code == code
    with pytest.raises(b200.LZ4FrameError) as e:
        b200.decompress_frames_dev(src, len(want) - 1)
    assert e.value.code == -9
    for bad_src in (src.cpu(), src.to(torch.int32)):
        with pytest.raises(ValueError):
            b200.decompress_frames_dev(bad_src, 400000)
    for bad_out in (torch.empty(400000, dtype=torch.uint8), torch.empty(400000, dtype=torch.int16, device="cuda")):
        with pytest.raises(ValueError):
            b200.decompress_frames_dev(src, 400000, out=bad_out)
