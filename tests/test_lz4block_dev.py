"""b200lz4block_compress_dev / b200lz4block_decompress_dev: lz4-java's LZ4Block streams (LZ4BlockOutputStream /
LZ4BlockInputStream) written and read in device memory, many streams per call.  Every stream of the fast compressor must be
byte for byte the stream assembled here by LZ4BlockOutputStream's rules from this library's block compressor at the same
source phase (_expected_stream), and the reader must return, stream by stream, what the restated LZ4BlockInputStream and the
host reader (b200lz4block_decompress_host) return.  Runs on the H100, and on the CPU emulator build of the library
(B200LZ4_TEST_SO=.../libb200lz4_sim.so), where the sizes shrink and torch is not used."""
import ctypes
import os
import random

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SIM = "sim" in os.environ.get("B200LZ4_TEST_SO", "")
E_ARG = -2147483645
SEED = 0x9747B28C
END_GUARD = 0xAA


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
            return arr.view(np.uint8).reshape(-1).copy()
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


def _u64(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.uint64).reshape(-1))


def _aligned(data: bytes, phase=0):
    """the bytes in a numpy buffer that starts `phase` bytes past a 64-byte boundary"""
    raw = np.empty(len(data) + 128, dtype=np.uint8)
    o = (-raw.ctypes.data) % 64 + phase
    a = raw[o:o + len(data)]
    a[:] = np.frombuffer(data, dtype=np.uint8)
    return a


def _lay_out(datas, align=64, phase=0, gap=0):
    """one source holding every stream's bytes at offsets = phase (mod align), `gap` bytes at least between them"""
    offs, pos = [], phase
    for d in datas:
        offs.append(pos)
        pos = (pos + len(d) + gap + align - 1) // align * align + phase
    src = np.zeros(pos + 64, dtype=np.uint8)
    for o, d in zip(offs, datas):
        src[o:o + len(d)] = np.frombuffer(d, dtype=np.uint8)
    return src, _u64(offs), _u64([len(d) for d in datas])


def _level(bs):
    return max(0, (bs - 1).bit_length() - 10)                         # LZ4BlockOutputStream.java:58-70


def _header(method, level, clen, olen, check):
    return b"LZ4Block" + bytes([method | level]) + clen.to_bytes(4, "little") + olen.to_bytes(4, "little") + check.to_bytes(4, "little")


def _expected_stream(b200, port, data, bs, phase=0):
    """the stream LZ4BlockOutputStream writes for `data` (LZ4BlockOutputStream.java:203-266), its blocks compressed by this
    library's fast block compressor as the writer runs it: one batch over the stream's blocks at the source's 16-byte phase,
    compressBound capacity each, max_src_len 65536 for blocks up to 64 KiB"""
    lvl, out = _level(bs), bytearray()
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
            block = data[o:o + n]
            stored = c <= 0 or c >= n
            payload = block if stored else comp[co:co + c].tobytes()
            out += _header(0x10 if stored else 0x20, lvl, len(payload), n, port.xxh32(block, SEED) & 0x0FFFFFFF) + payload
    return bytes(out + _header(0x10, lvl, 0, 0, 0))


def _check_layout(port, stream, data, bs):
    """what any LZ4BlockOutputStream writes for `data`, whatever its compressor: blocks of bs bytes, their checksums, the end block"""
    lvl, pos = _level(bs), 0
    for o in range(0, len(data), bs):
        block = data[o:o + bs]
        h = stream[pos:pos + 21]
        clen, olen = int.from_bytes(h[9:13], "little"), int.from_bytes(h[13:17], "little")
        assert h[:8] == b"LZ4Block" and h[8] & 0x0F == lvl and olen == len(block), (o, h)
        assert int.from_bytes(h[17:21], "little") == port.xxh32(block, SEED) & 0x0FFFFFFF, o
        assert (h[8] & 0xF0 == 0x10) == (clen == olen) and clen <= olen, o
        pos += 21 + clen
    assert stream[pos:] == _header(0x10, lvl, 0, 0, 0)


def _write(L, M, d_src, offs, lens, bs, hc=0, d_dst=None, cap=None, stream=None):
    """one b200lz4block_compress_dev call -> (rc, d_dst, stream_off, stream_len)"""
    if cap is None:
        cap = sum(L.b200lz4block_compress_bound(int(n), bs) for n in lens)
    if d_dst is None:
        d_dst = M.full(cap + 64, END_GUARD)
    so, sl = np.zeros(len(lens), dtype=np.uint64), np.zeros(len(lens), dtype=np.uint64)
    rc = L.b200lz4block_compress_dev(M.ptr(d_src), offs.ctypes.data, lens.ctypes.data, len(lens), M.ptr(d_dst), cap,
                                     so.ctypes.data, sl.ctypes.data, bs, hc, stream)
    return rc, d_dst, so, sl


def _read(L, M, d_src, offs, lens, d_dst, doff, dcap, stop, stream=None, result=True):
    """one b200lz4block_decompress_dev call -> (rc, result, src_consumed, content_len)"""
    ns = len(lens)
    res, used, content = np.zeros(ns, dtype=np.int64), np.zeros(ns, dtype=np.uint64), np.zeros(ns, dtype=np.uint64)
    rc = L.b200lz4block_decompress_dev(M.ptr(d_src), offs.ctypes.data, lens.ctypes.data, ns, M.ptr(d_dst), doff.ctypes.data,
                                       dcap.ctypes.data, int(stop), res.ctypes.data if result else None, used.ctypes.data,
                                       content.ctypes.data, stream)
    return rc, res, used, content


def _host_read(L, blob, cap, stop):
    """b200lz4block_decompress_host -> (result, src_consumed (0 unless result >= 0), bytes)"""
    src = np.frombuffer(bytes(blob) + bytes(64), dtype=np.uint8)
    dst = np.zeros(max(cap, 1), dtype=np.uint8)
    used = ctypes.c_size_t(0)
    r = L.b200lz4block_decompress_host(src.ctypes.data, len(blob), dst.ctypes.data, cap, int(stop), ctypes.byref(used))
    return r, (used.value if r >= 0 else 0), dst[:max(r, 0)].tobytes()


def _stream_datas(port, bs, rng):
    rdg = port.datagen(4 * bs + 4096, 0.5, 0.0, bs % 97).tobytes()
    lens = [0, 1, bs - 1, bs, bs + 1, 3 * bs + 17, rng.randrange(1, 4 * bs)]
    datas = []
    for k, n in enumerate(lens):
        kinds = (rdg[:n], rng.randbytes(n), bytes(n))                  # compressible, stored blocks, zeros
        datas += [kinds[k % 3]] if SIM else list(kinds)                # (the emulator runs ~30 ms per block)
    return datas


def _block_sizes():
    return (64, 1000, 4096, 65537) if SIM else (64, 1000, 4096, 32768, 65536, 65537, 1 << 20)


def test_writer_layout_and_read_back(b200, port):
    """every block size, stream lengths 0, 1, bs-1, bs, bs+1, 3bs+17 and one random, of RDG P=0.5, random bytes and zeros, all
    in one call per block size: each stream of the fast compressor is the expected one, HC level 9 streams have the layout
    and checksums LZ4BlockOutputStream writes (the HC kernel is not byte-identical from call to call), stream_off is
    contiguous from 0, and every stream reads back through the restated LZ4BlockInputStream and the host reader"""
    L, M = b200._native.lib(), _DevMem()
    rng = random.Random(1)
    for bs in _block_sizes():
        datas = _stream_datas(port, bs, rng)
        src, offs, lens = _lay_out(datas)
        d_src = M.up(src)
        for hc in ((0, 9) if not SIM or bs == 1000 else (0,)):
            rc, d_dst, so, sl = _write(L, M, d_src, offs, lens, bs, hc)
            assert rc == int(sl.sum()) and int(so[0]) == 0 and (so[1:] == so[:-1] + sl[:-1]).all(), (bs, hc, rc)
            out = M.down(d_dst)
            assert (out[rc:] == END_GUARD).all(), (bs, hc)                      # nothing past the total
            for k, d in enumerate(datas):
                s = out[int(so[k]):int(so[k] + sl[k])].tobytes()
                if hc == 0:
                    assert s == _expected_stream(b200, port, d, bs), (bs, k, len(d))
                else:
                    _check_layout(port, s, d, bs)
                assert port.lz4block_decompress(s, len(d)) == (len(d), d), (bs, hc, k)
                assert b200.decompress_lz4block(s, len(d)) == d, (bs, hc, k)


def test_host_writer_equals_the_device_writer_at_every_phase(b200, port):
    """b200lz4block_compress_host_hc (compress_lz4block) stages its source at the source's own 16-byte phase, so at each of the
    16 phases it writes what compress_lz4block_dev writes for the same bytes at that phase"""
    L, M = b200._native.lib(), _DevMem()
    data = port.datagen(70000 if SIM else 400000, 0.5, 0.0, 13).tobytes()
    streams = set()
    for p in range(16):
        src = np.zeros(len(data) + 64, dtype=np.uint8)
        src[p:p + len(data)] = np.frombuffer(data, dtype=np.uint8)
        rc, d_dst, _, _ = _write(L, M, M.up(src), _u64([p]), _u64([len(data)]), 65536)
        dev = M.down(d_dst)[:rc].tobytes()
        assert b200.compress_lz4block(_aligned(data, p), 65536) == dev, p
        streams.add(dev)
    assert len(streams) > 1                                                     # the phases chosen give different streams


def _faulty_streams(port, rng, n):
    """(blob, cap) pairs: the fault recipe of the host reader's sweep, concatenated streams, a stream without its end block
    followed by another (what syncFlush leaves), empty ranges, garbage"""
    base = port.datagen(1 << 18, 0.5, 0.0, 21).tobytes()

    def body():
        sizes = (1, 40, 700, 5000) if SIM else (1, 40, 700, 5000, 70000)
        b = b"".join(base[o:o + k] for o, k in ((rng.randrange(0, 100000), rng.choice(sizes)) for _ in range(rng.randrange(0, 4))))
        return b + (rng.randbytes(3000) if rng.random() < 0.2 else b"")

    out = []
    for _ in range(n):
        kind = rng.randrange(10)
        a = body()
        blob = bytearray(port.lz4block_compress(a, rng.choice((1024, 4096) if SIM else (64, 4096, 65536))))
        if kind == 0:
            blob += port.lz4block_compress(body(), 4096)                         # concatenated
        elif kind == 1:
            blob = blob[:-21] + port.lz4block_compress(body(), 4096)              # no end block, then another stream
        elif kind == 2:
            blob = bytearray()                                                    # an empty range
        elif kind == 3:
            blob += b"trailing bytes"
        if kind >= 3:
            for _ in range(rng.randrange(0, 4)):
                if rng.randrange(3) == 0 and len(blob) > 1:
                    del blob[rng.randrange(1, len(blob)):]
                elif blob:
                    i = rng.randrange(len(blob)); blob[i] ^= 1 << rng.randrange(8)
        full = max(port.lz4block_decompress(bytes(blob), 1 << 22, False)[0], port.lz4block_decompress(bytes(blob), 1 << 22, True)[0], len(a))
        cap = rng.choice((full, full, full + 8, full - 1000, 0))
        out.append((bytes(blob), max(cap, 0)))
    return out


def _read_all(L, M, cases, stop, caps=None):
    """every case in ONE device call, dst ranges with guard bytes between them -> (results, consumed, content, dst, doff)"""
    blobs = [b for b, _ in cases]
    caps = [c for _, c in cases] if caps is None else caps
    src, offs, lens = _lay_out(blobs, align=16, phase=3, gap=5)
    doff, pos = [], 7
    for c in caps:
        doff.append(pos)
        pos += int(c) + 24
    d_src, d_dst = M.up(src), M.full(pos + 64, END_GUARD)
    rc, res, used, content = _read(L, M, d_src, offs, lens, d_dst, _u64(doff), _u64(caps), stop)
    assert rc == 0, rc
    return res, used, content, M.down(d_dst), doff


def test_reader_parity_with_faults_in_one_call(b200, port):
    """hundreds of streams, truncated and bit-flipped, concatenated, without end blocks, empty, with capacities exact / +8 /
    -1000 / 0, read in one call for both stopOnEmptyBlock values: every stream's result and src_consumed are the restated
    LZ4BlockInputStream's and the host reader's, so is the content on success, and nothing outside a stream's range (nor,
    on success, past its result) is written.  content_len: every -9 stream read again with dst_cap = content_len gives no -9."""
    L, M = b200._native.lib(), _DevMem()
    rng = random.Random(2024)
    cases = _faulty_streams(port, rng, 40 if SIM else 600)
    seen = {}
    for stop in (True, False):
        res, used, content, dst, doff = _read_all(L, M, cases, stop)
        for k, (blob, cap) in enumerate(cases):
            want, out = port.lz4block_decompress(blob, cap, stop)
            h, h_used, h_out = _host_read(L, blob, cap, stop)
            assert int(res[k]) == want == h, (stop, k, int(res[k]), want, h)
            assert int(used[k]) == h_used, (stop, k)
            got = dst[doff[k]:doff[k] + cap]
            if want >= 0:
                assert int(content[k]) == want and got[:want].tobytes() == out == h_out, (stop, k)
                assert (got[want:] == END_GUARD).all(), (stop, k)
            assert (dst[doff[k] + cap:doff[k] + cap + 24] == END_GUARD).all(), (stop, k)
            seen[want if want < 0 else "ok"] = seen.get(want if want < 0 else "ok", 0) + 1
        assert (dst[:doff[0]] == END_GUARD).all()
        again = [k for k in range(len(cases)) if res[k] == -9]
        if again:
            res2, _, _, _, _ = _read_all(L, M, [cases[k] for k in again], stop, caps=[int(content[k]) for k in again])
            assert (res2 != -9).all(), (stop, res2)
    assert {"ok", -1, -2, -9} <= set(seen), seen


def test_reader_round_trip_with_the_writer(b200, port):
    """compress_dev -> decompress_dev over many streams at every block size: the sources come back, src_consumed is each
    stream's length, content_len its source length"""
    L, M = b200._native.lib(), _DevMem()
    rng = random.Random(5)
    for bs in _block_sizes():
        datas = _stream_datas(port, bs, rng)
        src, offs, lens = _lay_out(datas, align=16, phase=5)
        rc, d_streams, so, sl = _write(L, M, M.up(src), offs, lens, bs)
        assert rc > 0
        caps = lens
        d_dst = M.full(int(lens.sum()) + 64, END_GUARD)
        doff = _u64(np.cumsum(lens) - lens)
        r, res, used, content = _read(L, M, d_streams, so, sl, d_dst, doff, caps, True)
        out = M.down(d_dst)
        assert r == 0 and (res == lens.astype(np.int64)).all() and (used == sl).all() and (content == lens).all(), bs
        assert out[:int(lens.sum())].tobytes() == b"".join(datas) and (out[int(lens.sum()):] == END_GUARD).all(), bs


@pytest.mark.skipif(SIM, reason="2 GiB of device memory: GPU only")
def test_device_round_trip_at_scale(b200, port):
    """about 2 GiB in 4096 streams of mixed sizes, written and read back at 32 KiB, 64 KiB and 1 MiB blocks: every stream's
    XXH64 is its source's"""
    import torch
    L, M = b200._native.lib(), _DevMem()
    rng = np.random.default_rng(7)
    lens = rng.integers(0, 1 << 20, 4096).astype(np.uint64)
    lens[::97] = 0
    offs = _u64(np.cumsum(lens) - lens)
    total = int(lens.sum())
    piece = torch.from_numpy(port.datagen(64 << 20, 0.5, 0.0, 3)).cuda()
    d_src = piece.repeat(total // piece.numel() + 1)[:total + 64].contiguous()
    d_src[-64:] = 0
    del piece

    def xxh64(buf, o, n):
        out = torch.zeros(len(n), dtype=torch.int64, device="cuda")
        b200.batch.xxh64_batch_dev(buf, torch.from_numpy(o.astype(np.int64)).cuda(), torch.from_numpy(n.astype(np.int32)).cuda(), out)
        return out.cpu().numpy()

    want = xxh64(d_src, offs, lens)
    d_out = torch.full((total + 64,), END_GUARD, dtype=torch.uint8, device="cuda")
    for bs in (32768, 65536, 1 << 20):
        streams, so, sl = b200.compress_lz4block_dev(d_src, offs, lens, block_size=bs)
        res, used, content = b200.decompress_lz4block_dev(streams, so, sl, d_out, offs, lens)
        assert (res == lens.astype(np.int64)).all() and (used == sl).all() and (content == lens).all(), bs
        assert (xxh64(d_out, offs, lens) == want).all(), bs
        assert (d_out[total:] == END_GUARD).all()
        del streams


def test_errors_launch_nothing_and_write_nothing(b200, port):
    """writer: dst_capacity one short of the bounds (-9), blockSize 63 and 32 MiB + 1 (B200LZ4_E_ARG), no streams (0);
    reader: a NULL result array, NULL offsets, a destination range that overflows (B200LZ4_E_ARG; the stream is only its end
    block, so nothing would be written), no streams (0): no launch, no byte written"""
    L, M = b200._native.lib(), _DevMem()
    datas = [port.datagen(100000, 0.5, 0.0, 6).tobytes(), b"xyz"]
    src, offs, lens = _lay_out(datas)
    d_src = M.up(src)
    cap = sum(L.b200lz4block_compress_bound(int(n), 65536) for n in lens)
    d_dst = M.full(cap + 64, END_GUARD)
    before = L.b200lz4_launch_count()
    assert _write(L, M, d_src, offs, lens, 65536, d_dst=d_dst, cap=cap - 1)[0] == -9
    for bs in (63, (1 << 25) + 1):
        assert _write(L, M, d_src, offs, lens, bs, d_dst=d_dst, cap=cap + 64)[0] == E_ARG, bs
    assert _write(L, M, d_src, offs[:0], lens[:0], 65536, d_dst=d_dst, cap=cap)[0] == 0
    doff, dcap = _u64([0, 100000]), _u64([100000, 3])
    assert _read(L, M, d_src, offs, lens, d_dst, doff, dcap, True, result=False)[0] == E_ARG
    assert L.b200lz4block_decompress_dev(M.ptr(d_src), None, lens.ctypes.data, 2, M.ptr(d_dst), doff.ctypes.data, dcap.ctypes.data,
                                         1, np.zeros(2, dtype=np.int64).ctypes.data, None, None, None) == E_ARG
    d_end = M.up(np.frombuffer(_header(0x10, 0, 0, 0, 0), dtype=np.uint8))
    assert _read(L, M, d_end, _u64([0]), _u64([21]), d_dst, _u64([2**64 - 2]), _u64([16]), True)[0] == E_ARG
    assert _read(L, M, d_src, offs[:0], lens[:0], d_dst, doff[:0], dcap[:0], True)[0] == 0
    assert L.b200lz4_launch_count() == before
    assert (M.down(d_dst) == END_GUARD).all()


def test_launches_do_not_depend_on_streams(b200, port):
    """the same bytes as 1, 64 and 4096 streams (1, 16 and 64 of 64 blocks on the emulator; equal blocks, same phases): the
    writer and the reader launch the same kernels"""
    L, M = b200._native.lib(), _DevMem()
    bs, nb = (256, 64) if SIM else (4096, 4096)
    data = port.datagen(nb * bs, 0.5, 0.0, 7).tobytes()
    counts = []
    for ns in ((1, 16, 64) if SIM else (1, 64, 4096)):
        per = len(data) // ns
        offs, lens = _u64(np.arange(ns) * per), _u64([per] * ns)
        d_src = M.up(np.frombuffer(data + bytes(64), dtype=np.uint8))
        before = L.b200lz4_launch_count()
        rc, d_streams, so, sl = _write(L, M, d_src, offs, lens, bs)
        mid = L.b200lz4_launch_count()
        d_dst = M.full(len(data) + 64, END_GUARD)
        r, res, _, _ = _read(L, M, d_streams, so, sl, d_dst, offs, lens, True)
        counts.append((mid - before, L.b200lz4_launch_count() - mid))
        assert rc > 0 and r == 0 and (res == per).all() and M.down(d_dst)[:len(data)].tobytes() == data, ns
    assert counts[0] == counts[1] == counts[2], counts


@pytest.mark.skipif(not SIM, reason="the counting emulator build counts the library's host<->device copies")
def test_no_payload_crosses_to_the_host(b200, port):
    """two calls with the same streams and blocks whose payloads differ 64x in size: the writer and the reader copy the same
    bytes between host and device for both, a small constant per block and per stream (on the counting emulator library,
    tests/simt/copy_count.h, which test_lz4block_sim.py builds)"""
    L, M = b200._native.lib(), _DevMem()
    if not hasattr(L, "b200lz4_sim_copied_bytes"):
        pytest.skip("this emulator library does not count copies: tests/simt/copy_count.h")
    L.b200lz4_sim_copied_bytes.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
    h2d, d2h = ctypes.c_ulonglong(0), ctypes.c_ulonglong(0)

    def copied(fn):
        L.b200lz4_sim_copied_bytes(ctypes.byref(h2d), ctypes.byref(d2h))
        a = (h2d.value, d2h.value)
        fn()
        L.b200lz4_sim_copied_bytes(ctypes.byref(h2d), ctypes.byref(d2h))
        return h2d.value - a[0], d2h.value - a[1]

    rng = random.Random(8)
    counts = {"write": [], "read": []}
    for bs in (1024, 65536):
        datas = [rng.randbytes(4 * bs) for _ in range(8)]                      # 8 streams of 4 stored blocks each
        src, offs, lens = _lay_out(datas)
        d_src = M.up(src)
        got = {}
        counts["write"].append(copied(lambda: got.update(w=_write(L, M, d_src, offs, lens, bs))))
        rc, d_streams, so, sl = got["w"]
        d_dst = M.full(int(lens.sum()) + 64, 0)
        doff = _u64(np.cumsum(lens) - lens)
        counts["read"].append(copied(lambda: got.update(r=_read(L, M, d_streams, so, sl, d_dst, doff, lens, True))))
        assert got["r"][0] == 0 and (got["r"][1] == 4 * bs).all()
    for fn, c in counts.items():
        assert c[0] == c[1], (fn, c)
        assert 0 < c[0][0] and 0 < c[0][1] and sum(c[0]) < 8 * 4 * 1024, (fn, c)


@pytest.mark.skipif(SIM, reason="torch streams: GPU only")
def test_ordered_after_a_side_stream(b200, port):
    """the sources are written by torch ops on a side stream and both calls are made on that stream without a synchronise:
    the streams hold the new bytes and decode to them"""
    import torch
    old, new = port.datagen(4 << 20, 0.5, 0.0, 1), port.datagen(4 << 20, 0.5, 0.0, 2)
    offs, lens = _u64([0, 3 << 20]), _u64([3 << 20, 1 << 20])
    d_src, d_new = torch.from_numpy(old.copy()).cuda(), torch.from_numpy(new.copy()).cuda()
    d_out = torch.zeros(4 << 20, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.cuda._sleep(20_000_000)                                       # the copy lands well after the call is made
        d_src.copy_(d_new)
        streams, so, sl = b200.compress_lz4block_dev(d_src, offs, lens)
        copy = torch.zeros_like(streams)
        torch.cuda._sleep(20_000_000)
        copy.copy_(streams)                                                 # the reader's input lands well after the call too
        res, _, _ = b200.decompress_lz4block_dev(copy, so, sl, d_out, offs, lens)
    torch.cuda.synchronize()
    host = streams.cpu().numpy()
    for k in range(2):
        s = host[int(so[k]):int(so[k] + sl[k])].tobytes()
        assert s == _expected_stream(b200, port, new[int(offs[k]):int(offs[k] + lens[k])].tobytes(), 1 << 16), k
    assert (res == lens.astype(np.int64)).all() and d_out.cpu().numpy().tobytes() == new.tobytes()


@pytest.mark.skipif(SIM, reason="torch tensors: GPU only")
def test_python_wrappers(b200, port):
    import torch
    datas = [port.datagen(300000, 0.5, 0.0, 9).tobytes(), b"", b"abc"]
    src, offs, lens = _lay_out(datas)
    d_src = torch.from_numpy(src).cuda()
    streams, so, sl = b200.compress_lz4block_dev(d_src, list(offs), list(lens), block_size=4096)
    assert streams.is_cuda and so.dtype == np.uint64 and sl.dtype == np.uint64
    host = streams.cpu().numpy()
    for k, d in enumerate(datas):
        assert host[int(so[k]):int(so[k] + sl[k])].tobytes() == b200.compress_lz4block(_aligned(d), 4096), k
    out = torch.full((400000,), END_GUARD, dtype=torch.uint8, device="cuda")
    bound = sum(b200._native.lib().b200lz4block_compress_bound(int(n), 4096) for n in lens)
    w = torch.full((bound + 100,), END_GUARD, dtype=torch.uint8, device="cuda")
    got, _, _ = b200.compress_lz4block_dev(d_src, offs, lens, 4096, out=w)
    assert got.data_ptr() == w.data_ptr() and (w[got.numel():] == END_GUARD).all()
    doff = [0, 300000, 300100]
    res, used, content = b200.decompress_lz4block_dev(streams, so, sl, out, doff, [300000, 10, 2], stop_on_empty_block=False)
    assert res.dtype == np.int64 and res.tolist() == [300000, 0, -9] and content.tolist() == [300000, 0, 3]
    assert used.tolist() == [int(sl[0]), int(sl[1]), 0]
    assert out[:300000].cpu().numpy().tobytes() == datas[0]
    with pytest.raises(ValueError):
        b200.compress_lz4block_dev(d_src, offs, lens, block_size=63)
    with pytest.raises(ValueError):
        b200.compress_lz4block_dev(d_src.cpu(), offs, lens)
    with pytest.raises(ValueError):
        b200.compress_lz4block_dev(d_src, offs, [len(src) + 1, 0, 0])
    with pytest.raises(b200.LZ4FrameError) as e:
        b200.compress_lz4block_dev(d_src, offs, lens, out=torch.empty(10, dtype=torch.uint8, device="cuda"))
    assert e.value.code == -9
    with pytest.raises(ValueError):
        b200.decompress_lz4block_dev(streams, so, sl, out.cpu(), doff, [1, 1, 1])
    with pytest.raises(ValueError):
        b200.decompress_lz4block_dev(streams, so, sl, out, doff, [1, 1])
    with pytest.raises(ValueError):
        b200.decompress_lz4block_dev(streams, so, sl, out, doff, [1, 1, 400000])
