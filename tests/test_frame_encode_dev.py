"""b200lz4f_compress_dev: LZ4 frames of device-resident bytes, written on the device, and b200lz4f_compress_host_hc, the same
writer on a device copy of a host source.  Every frame of the fast compressor must be byte for byte the frame assembled here
by LZ4FrameOutputStream's rules from this library's block compressor at the same source phase (_expected_frame), and every
frame must be read back by this library's frame reader, the restated LZ4FrameInputStream and the reference's LZ4F_decompress.
Runs on the H100, and on the CPU emulator build of the library (B200LZ4_TEST_SO=.../libb200lz4_sim.so), where the sizes
shrink and torch is not used."""
import os
import random

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SIM = "sim" in os.environ.get("B200LZ4_TEST_SO", "")
E_ARG = -2147483645


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


def _aligned(data: bytes, phase=0):
    """the bytes in a numpy buffer that starts `phase` bytes past a 64-byte boundary"""
    raw = np.empty(len(data) + 128, dtype=np.uint8)
    o = (-raw.ctypes.data) % 64 + phase
    a = raw[o:o + len(data)]
    a[:] = np.frombuffer(data, dtype=np.uint8)
    return a


def _lay_out(datas, align=64, phase=0):
    """one device source holding every frame's bytes at offsets = phase (mod align)"""
    offs, pos = [], phase
    for d in datas:
        offs.append(pos)
        pos = (pos + len(d) + align - 1) // align * align + phase
    src = np.zeros(pos + 64, dtype=np.uint8)
    for o, d in zip(offs, datas):
        src[o:o + len(d)] = np.frombuffer(d, dtype=np.uint8)
    return src, np.asarray(offs, dtype=np.uint64), np.asarray([len(d) for d in datas], dtype=np.uint64)


def _bound(L, lens, bs_code):
    return sum(L.b200lz4f_compress_bound(int(n), bs_code) for n in lens)


def _write(L, M, d_src, offs, lens, bs_code, flags, hc=0, d_dst=None, cap=None, stream=None):
    """one b200lz4f_compress_dev call -> (rc, d_dst, frame_off, frame_len)"""
    if cap is None:
        cap = _bound(L, lens, bs_code)
    if d_dst is None:
        d_dst = M.full(cap + 64, 0)
    fo, fl = np.zeros(len(lens), dtype=np.uint64), np.zeros(len(lens), dtype=np.uint64)
    rc = L.b200lz4f_compress_dev(M.ptr(d_src), offs.ctypes.data, lens.ctypes.data, len(lens), M.ptr(d_dst), cap,
                                 fo.ctypes.data, fl.ctypes.data, bs_code, flags, hc, stream)
    return rc, d_dst, fo, fl


def _frames(out, fo, fl):
    return [out[int(o):int(o) + int(n)].tobytes() for o, n in zip(fo, fl)]


def _expected_frame(b200, port, data, bs_code, flags, phase=0):
    """the frame LZ4FrameOutputStream writes for `data` (LZ4FrameOutputStream.java:178-251), its blocks compressed by this
    library's fast block compressor as the frame writer runs it: one batch over the frame's blocks at the source's 16-byte
    phase, compressBound capacity each, max_src_len 65536 for 64 KiB blocks (GPU streams are not the CPU restatement's)"""
    flg = 0x60 | (0x10 if flags & 2 else 0) | (0x08 if flags & 4 else 0) | (0x04 if flags & 1 else 0)
    desc = bytes([flg, bs_code << 4]) + (len(data).to_bytes(8, "little") if flags & 4 else b"")
    out = bytearray(b"\x04\x22\x4d\x18" + desc + bytes([(port.xxh32(desc, 0) >> 8) & 0xFF]))
    bs = 1 << (8 + 2 * bs_code)
    if data:
        offs = np.arange(0, len(data), bs, dtype=np.uint64)
        lens = np.minimum(bs, len(data) - offs).astype(np.int32)
        cap = lens + lens // 255 + 16
        slot = (cap.astype(np.uint64) + 15) // 16 * 16
        coff = np.cumsum(slot) - slot
        comp = np.zeros(int(slot.sum()), dtype=np.uint8)
        clen = b200.batch.compress_fast_batch_host(_aligned(data, phase), offs, lens, comp, coff, cap,
                                                   max_src_len=65536 if bs <= 65536 else 0)
        for o, n, co, c in zip(offs.tolist(), lens.tolist(), coff.tolist(), clen.tolist()):
            stored = c <= 0 or c >= n                                   # (:215-222)
            payload = data[o:o + n] if stored else comp[co:co + c].tobytes()
            out += (len(payload) | (0x80000000 if stored else 0)).to_bytes(4, "little") + payload
            if flags & 2:
                out += port.xxh32(payload, 0).to_bytes(4, "little")
    out += bytes(4)                                                     # EndMark
    if flags & 1:
        out += port.xxh32(data, 0).to_bytes(4, "little")
    return bytes(out)


def _reference():
    from oracle import oracle as O
    try:
        return O.Ref()
    except (FileNotFoundError, OSError):
        return None


def _check_readers(b200, port, ref, frames, datas, whole=None):
    if whole is not None:
        assert b200.decompress_frames(whole, sum(map(len, datas)) + 8) == b"".join(datas)
    for f, d in zip(frames, datas):
        assert port.frame_decompress(f, len(d) + 8) == (len(d), d)
        if ref is not None:
            assert ref.frame_decompress(f, len(d) + 8) == (len(d), d), "LZ4F_decompress"


def _mixed(port):
    rng = random.Random(11)
    rdg = port.datagen(1 << 20, 0.5, 0.0, 3).tobytes()
    sizes = (0, 1, 100, 65535, 65536, 65537, 300000) if SIM else (0, 1, 100, 65535, 65536, 65537, 300000, 3 * (1 << 20) + 5)
    datas = [(rdg * 4)[:n] for n in sizes]
    datas.append(rng.randbytes(200000))                                  # does not shrink: stored blocks
    datas.append(port.datagen(150000 if SIM else 1500000, 0.5, 0.0, 8).tobytes())
    return datas


def test_frames_equal_the_host_writer_and_every_reader_reads_them(b200, port):
    """every bsCode 4..7 and flags 0..7 over one mixed call at 64-byte-aligned device offsets: each frame is the expected
    one, frame_off is contiguous from 0, the return value is the sum of frame_len, and the frames decode with this
    library's reader (all of them at once), the restated LZ4FrameInputStream and the reference's LZ4F_decompress"""
    L, M, ref = b200._native.lib(), _DevMem(), _reference()
    datas = _mixed(port)
    src, offs, lens = _lay_out(datas)
    d_src = M.up(src)
    combos = [(bs, fl) for bs in (4, 5, 6, 7) for fl in range(8)]
    if SIM:
        combos = [(4, 0), (4, 7), (5, 3), (6, 5), (7, 6), (7, 1)]
    for bs, fl in combos:
        rc, d_dst, fo, fl_ = _write(L, M, d_src, offs, lens, bs, fl)
        assert rc == int(fl_.sum()), (bs, fl, rc)
        assert int(fo[0]) == 0 and (fo[1:] == fo[:-1] + fl_[:-1]).all(), (bs, fl)
        out = M.down(d_dst)
        frames = _frames(out, fo, fl_)
        for k, (f, d) in enumerate(zip(frames, datas)):
            assert f == _expected_frame(b200, port, d, bs, fl), (bs, fl, k, len(d))
        _check_readers(b200, port, ref, frames, datas, out[:rc].tobytes())


def test_unaligned_sources_give_valid_frames(b200, port):
    """sources at offsets 1, 2, 3 and 7 (mod 16): the compressor may parse differently there (DESIGN.md §4, source
    alignment), so the frames need not be those of 16-byte-aligned sources, but they are valid and decode to their input"""
    L, M, ref = b200._native.lib(), _DevMem(), _reference()
    data = port.datagen(200000 if SIM else 2000000, 0.5, 0.0, 4).tobytes()
    datas = [data[:n] for n in (70000, 1, 0, 150000 if SIM else 1500000, 65536)]
    for phase in (1, 2, 3, 7):
        src, offs, lens = _lay_out(datas, align=16, phase=phase)
        for bs, fl in ((4, 7), (5, 2)):
            rc, d_dst, fo, fl_ = _write(L, M, M.up(src), offs, lens, bs, fl)
            assert rc == int(fl_.sum()), (phase, bs, fl)
            out = M.down(d_dst)
            _check_readers(b200, port, ref, _frames(out, fo, fl_), datas, out[:rc].tobytes())


def test_high_compressor_frames(b200, port):
    """hc_level 3, 9, 12: readable by every reader and no larger than the fast compressor's frames on compressible data
    (not byte-identical from call to call: the HC kernel's ring insert order comes from atomicAdd)"""
    L, M, ref = b200._native.lib(), _DevMem(), _reference()
    datas = [port.datagen(n, 0.5, 0.0, 5 + n % 7).tobytes() for n in ((70000, 1) if SIM else (300000, 65537, 1, 0, 1500000))]
    src, offs, lens = _lay_out(datas)
    d_src = M.up(src)
    _, d_fast, fo_f, fl_f = _write(L, M, d_src, offs, lens, 4, 7)
    for level in ((9,) if SIM else (3, 9, 12)):
        rc, d_dst, fo, fl_ = _write(L, M, d_src, offs, lens, 4, 7, hc=level)
        assert rc == int(fl_.sum()), level
        out = M.down(d_dst)
        _check_readers(b200, port, ref, _frames(out, fo, fl_), datas, out[:rc].tobytes())
        assert (fl_ <= fl_f).all(), (level, fl_, fl_f)


def test_calls_that_span_several_chunks(b200, port):
    """a call cut into several internal chunks (CHUNK_SPAN, B200LZ4_CHUNK_MB) is the expected one, frame by frame: the
    running offset is carried from chunk to chunk on the device"""
    L, M = b200._native.lib(), _DevMem()
    total = (2 << 20) if SIM else (600 << 20)
    data = port.datagen(total, 0.5, 0.0, 12).tobytes()
    cuts = [0, total // 7, total // 7 + 1, total // 2 + 12345, total - 65536 * 3 - 9, total]
    datas = [data[a:b] for a, b in zip(cuts, cuts[1:])]
    src, offs, lens = _lay_out(datas)
    d_src = M.up(src)
    for bs, fl in ((4, 7), (7, 3)):
        rc, d_dst, fo, fl_ = _write(L, M, d_src, offs, lens, bs, fl)
        assert rc == int(fl_.sum()), (bs, fl)
        out = M.down(d_dst)
        for k, (f, d) in enumerate(zip(_frames(out, fo, fl_), datas)):
            assert f == _expected_frame(b200, port, d, bs, fl), (bs, fl, k)


def test_host_writer_keeps_the_source_phase(b200, port):
    """b200lz4f_compress_host_hc (compress_frame) stages the source at its own 16-byte phase before the device writer runs,
    so its frame is the expected one at that phase; the phases chosen give different frames for the longest source"""
    data = port.datagen(200000, 0.5, 0.0, 13).tobytes()
    sizes = (0, 1, 65536, 65537) if SIM else (0, 1, 100, 65536, 65537, 200000)
    for n in sizes:
        for fl in (0, 7):
            want = {p: _expected_frame(b200, port, data[:n], 4, fl, p) for p in (0, 1, 3, 8)}
            for p, w in want.items():
                got = b200.compress_frame(_aligned(data[:n], p), 4, bool(fl & 1), bool(fl & 2), bool(fl & 4))
                assert got == w, (n, fl, p)
    assert len(set(want.values())) > 1


@pytest.mark.skipif(SIM, reason="torch streams: GPU only")
def test_ordered_after_the_stream_and_nothing_written_past_the_frames(b200, port):
    """the source is written by a torch op on a side stream and the writer is called on that stream without a synchronise:
    the frames hold the new bytes, and d_dst past the frames still holds what was there"""
    import torch
    L, M = b200._native.lib(), _DevMem()
    old, new = port.datagen(4 << 20, 0.5, 0.0, 1), port.datagen(4 << 20, 0.5, 0.0, 2)
    datas = [new[:3 << 20].tobytes(), new[3 << 20:].tobytes()]
    offs, lens = np.asarray([0, 3 << 20], dtype=np.uint64), np.asarray([3 << 20, 1 << 20], dtype=np.uint64)
    d_src, d_new = M.up(old), M.up(new)
    cap = _bound(L, lens, 4)
    d_dst = M.full(cap + 4096, 0xAA)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        d_src.copy_(d_new)
        rc, _, fo, fl_ = _write(L, M, d_src, offs, lens, 4, 7, d_dst=d_dst, cap=cap + 4096, stream=side.cuda_stream)
    out = M.down(d_dst)
    assert rc == int(fl_.sum())
    for f, d in zip(_frames(out, fo, fl_), datas):
        assert f == _expected_frame(b200, port, d, 4, 7)
    assert (out[rc:] == 0xAA).all()


def test_errors_launch_nothing_and_write_nothing(b200, port):
    L, M = b200._native.lib(), _DevMem()
    datas = [port.datagen(100000, 0.5, 0.0, 6).tobytes(), b"xyz"]
    src, offs, lens = _lay_out(datas)
    d_src = M.up(src)
    cap = _bound(L, lens, 4)
    d_dst = M.full(cap + 64, 0xAA)
    before = L.b200lz4_launch_count()
    assert _write(L, M, d_src, offs, lens, 4, 7, d_dst=d_dst, cap=cap - 1)[0] == -9
    for bs in (3, 8):
        assert _write(L, M, d_src, offs, lens, bs, 7, d_dst=d_dst, cap=cap + 64)[0] == E_ARG, bs
    assert _write(L, M, d_src, offs[:0], lens[:0], 4, 7, d_dst=d_dst, cap=cap)[0] == 0
    assert L.b200lz4_launch_count() == before
    assert (M.down(d_dst) == 0xAA).all()


@pytest.mark.skipif(SIM, reason="2 GiB of device memory: GPU only")
def test_content_checksum_of_a_frame_past_2_gib_is_refused(b200):
    import torch
    L, M = b200._native.lib(), _DevMem()
    d_src = torch.zeros((1 << 31) + 1, dtype=torch.uint8, device="cuda")
    offs, lens = np.asarray([0], dtype=np.uint64), np.asarray([1 << 31], dtype=np.uint64)
    d_dst = M.full(4096, 0xAA)
    before = L.b200lz4_launch_count()
    cap = _bound(L, lens, 7)                       # only checked, never reached: the call fails before writing
    assert _write(L, M, d_src, offs, lens, 7, 1, d_dst=d_dst, cap=cap)[0] == -10
    assert L.b200lz4_launch_count() == before and (M.down(d_dst) == 0xAA).all()
    del d_src


def test_launches_depend_on_chunks_not_frames(b200, port):
    """one frame of 64 x 64 KiB and 64 frames of 64 KiB: the same launches"""
    L, M = b200._native.lib(), _DevMem()
    n = 8 if SIM else 64
    data = port.datagen(n * 65536, 0.5, 0.0, 7).tobytes()
    one = _lay_out([data])
    many = _lay_out([data[k * 65536:(k + 1) * 65536] for k in range(n)])
    for fl in (0, 7):
        counts = []
        for src, offs, lens in (one, many):
            d_src = M.up(src)
            before = L.b200lz4_launch_count()
            rc = _write(L, M, d_src, offs, lens, 4, fl)[0]
            assert rc > 0
            counts.append(L.b200lz4_launch_count() - before)
        assert counts[0] == counts[1], (fl, counts)


@pytest.mark.skipif(SIM, reason="torch tensors: GPU only")
def test_python_wrapper(b200, port):
    import torch
    L, M = b200._native.lib(), _DevMem()
    datas = [port.datagen(300000, 0.5, 0.0, 9).tobytes(), b"", b"abc"]
    src, offs, lens = _lay_out(datas)
    d_src = M.up(src)
    rc, d_dst, fo, fl_ = _write(L, M, d_src, offs, lens, 5, 6)
    want = M.down(d_dst)[:rc].tobytes()
    got, foff, flen = b200.compress_frames_dev(d_src, list(offs), list(lens), block_size_code=5, content_checksum=False,
                                               block_checksum=True, content_size=True)
    assert got.is_cuda and got.cpu().numpy().tobytes() == want
    assert foff.dtype == np.uint64 and (foff == fo).all() and (flen == fl_).all()
    out = torch.full((_bound(L, lens, 5) + 100,), 0xAA, dtype=torch.uint8, device="cuda")
    got2, _, _ = b200.compress_frames_dev(d_src, offs, lens, 5, False, True, True, out=out)
    assert got2.data_ptr() == out.data_ptr() and got2.cpu().numpy().tobytes() == want
    assert (out[rc:] == 0xAA).all()
    with pytest.raises(ValueError):
        b200.compress_frames_dev(d_src, offs, lens, block_size_code=3)
    with pytest.raises(b200.LZ4FrameError) as e:
        b200.compress_frames_dev(d_src, offs, lens, out=torch.empty(10, dtype=torch.uint8, device="cuda"))
    assert e.value.code == -9
