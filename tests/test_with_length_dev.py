"""b200lz4_compress_with_length_dev / b200lz4_decompress_with_length_dev: lz4-java's length-prefixed records
(LZ4CompressorWithLength / LZ4DecompressorWithLength: 4 bytes of little-endian original length, then one LZ4 block) written
and read in device memory, many records per call.  Every record of the fast compressor must be byte for byte what the host
call b200lz4_compress_with_length writes for the same bytes at the same 16-byte source phase, and the reader must return,
record by record, what the host calls b200lz4_decompress_with_length (fast flavour) and b200lz4_decompress_with_length_safe
(safe flavour) return.  Runs on the H100, and on the CPU emulator build of the library
(B200LZ4_TEST_SO=.../libb200lz4_sim.so), where the sizes shrink and torch is not used."""
import ctypes
import os
import random

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SIM = "sim" in os.environ.get("B200LZ4_TEST_SO", "")
E_ARG = -2147483645
END_GUARD = 0xAA
CHUNK_SPAN = int(os.environ.get("B200LZ4_CHUNK_MB", "256")) << 20


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
    """one source holding every record's bytes at offsets = phase (mod align), `gap` bytes at least between them"""
    offs, pos = [], phase
    for d in datas:
        offs.append(pos)
        pos = (pos + len(d) + gap + align - 1) // align * align + phase
    src = np.zeros(pos + 64, dtype=np.uint8)
    for o, d in zip(offs, datas):
        src[o:o + len(d)] = np.frombuffer(d, dtype=np.uint8)
    return src, _u64(offs), _u64([len(d) for d in datas])


def _lay_out_phases(datas):
    """one source holding record k at 16-byte phase k % 16"""
    offs, pos = [], 0
    for k, d in enumerate(datas):
        pos = (pos + 15) // 16 * 16 + k % 16
        offs.append(pos)
        pos += len(d)
    src = np.zeros(pos + 64, dtype=np.uint8)
    for o, d in zip(offs, datas):
        src[o:o + len(d)] = np.frombuffer(d, dtype=np.uint8)
    return src, _u64(offs), _u64([len(d) for d in datas])


def _bound(n):
    return n + n // 255 + 16 + 4


def _write(L, M, d_src, offs, lens, hc=0, d_dst=None, cap=None, stream=None):
    """one b200lz4_compress_with_length_dev call -> (rc, d_dst, rec_off, rec_len)"""
    if cap is None:
        cap = sum(_bound(int(n)) for n in lens)
    if d_dst is None:
        d_dst = M.full(cap + 64, END_GUARD)
    ro, rl = np.zeros(len(lens), dtype=np.uint64), np.zeros(len(lens), dtype=np.uint64)
    rc = L.b200lz4_compress_with_length_dev(M.ptr(d_src), offs.ctypes.data, lens.ctypes.data, len(lens), M.ptr(d_dst), cap,
                                            ro.ctypes.data, rl.ctypes.data, hc, stream)
    return rc, d_dst, ro, rl


def _read(L, M, d_src, offs, lens, d_dst, doff, dcap, safe, stream=None, result=True):
    """one b200lz4_decompress_with_length_dev call -> (rc, result, orig_len)"""
    n = len(lens)
    res, orig = np.zeros(n, dtype=np.int64), np.zeros(n, dtype=np.int64)
    rc = L.b200lz4_decompress_with_length_dev(M.ptr(d_src), offs.ctypes.data, lens.ctypes.data, n, M.ptr(d_dst),
                                              doff.ctypes.data, dcap.ctypes.data, int(safe),
                                              res.ctypes.data if result else None, orig.ctypes.data, stream)
    return rc, res, orig


def _host_record(L, data, phase):
    """b200lz4_compress_with_length on `data` at `phase`"""
    src, cap = _aligned(data, phase), _bound(len(data))
    dst = np.zeros(cap, dtype=np.uint8)
    r = L.b200lz4_compress_with_length(src.ctypes.data if len(data) else None, dst.ctypes.data, len(data), cap)
    assert r > 0, r
    return dst[:r].tobytes()


def _host_read(L, blob, cap, safe):
    """b200lz4_decompress_with_length{,_safe} -> (result, the bytes it decoded)"""
    src = np.frombuffer(bytes(blob) + bytes(64), dtype=np.uint8)
    dst = np.zeros(max(cap, 1), dtype=np.uint8)
    fn = L.b200lz4_decompress_with_length_safe if safe else L.b200lz4_decompress_with_length
    r = fn(src.ctypes.data, len(blob), dst.ctypes.data, cap)
    declared = int.from_bytes(blob[:4], "little", signed=True) if len(blob) >= 4 else -1
    return r, dst[:(r if safe else declared) if r >= 0 else 0].tobytes()


def _oracle_ref():
    from oracle import oracle as O
    try:
        return O.Ref()
    except (FileNotFoundError, OSError):
        return None


def _writer_datas(port, rng):
    """lengths 0, 1, 12, 13, 4096, 65535, 65536, 65537 and 1 MiB (not under the emulator) of RDG P=0.5, random bytes and
    zeros, and one record larger than a chunk, shuffled so that the two compressor classes alternate inside a chunk"""
    lens = [0, 1, 12, 13, 4096, 65535, 65536, 65537] + ([] if SIM else [1 << 20])
    rdg = port.datagen(max(lens) + 4096, 0.5, 0.0, 11).tobytes()
    datas = []
    for k, n in enumerate(lens):
        kinds = (rdg[:n], rng.randbytes(n), bytes(n))
        datas += [kinds[k % 3]] if SIM and n > 4096 else list(kinds)   # (the emulator runs one warp per block, slowly)
    rng.shuffle(datas)
    big = CHUNK_SPAN + 4097                                            # alone in its chunk, whatever the chunk size
    datas.insert(len(datas) // 2, rdg[:65536] + bytes(big - 65536))
    return datas


def test_writer_parity_with_the_host_call_at_every_phase(b200, port):
    """every record of the fast compressor is what b200lz4_compress_with_length writes for the same bytes at the same
    16-byte phase (records sit at all 16 phases, short and long ones alternating inside a chunk, one longer than a chunk),
    rec_off is contiguous from 0, nothing is written past the total, and every record decodes with the oracle and, where it
    is built, the reference's LZ4_decompress_safe"""
    L, M = b200._native.lib(), _DevMem()
    ref = _oracle_ref()
    datas = _writer_datas(port, random.Random(1))
    src, offs, lens = _lay_out_phases(datas)
    rc, d_dst, ro, rl = _write(L, M, M.up(src), offs, lens)
    assert rc == int(rl.sum()) and int(ro[0]) == 0 and (ro[1:] == ro[:-1] + rl[:-1]).all(), rc
    out = M.down(d_dst)
    assert (out[rc:] == END_GUARD).all()
    for k, d in enumerate(datas):
        rec = out[int(ro[k]):int(ro[k] + rl[k])].tobytes()
        assert rec == _host_record(L, d, int(offs[k]) % 16), (k, len(d))
        assert int.from_bytes(rec[:4], "little") == len(d)
        assert port.decompress_safe(rec[4:], len(d)) == (len(d), d), (k, len(d))
        if ref is not None:
            assert ref.decompress_safe(rec[4:], len(d)) == (len(d), d), (k, len(d))
    assert len({int(o) % 16 for o in offs}) == 16


def test_writer_hc_levels(b200, port):
    """hc_level 1, 4, 9, 12 (9 under the emulator): a record is the 4-byte length followed by an LZ4_compress_HC block of the
    record, which decodes to it as the block of b200lz4_compress_HC does, within the record bound.  The HC kernel's bytes are
    not compared: its ring insert order comes from atomicAdd, so they differ from call to call."""
    L, M = b200._native.lib(), _DevMem()
    rdg = port.datagen(70000, 0.5, 0.0, 12).tobytes()
    datas = [rdg[:n] for n in ((0, 1, 13, 4096) if SIM else (0, 1, 13, 4096, 65536, 65537, 70000))]
    src, offs, lens = _lay_out(datas, align=16, phase=7)
    d_src = M.up(src)
    for level in ((9,) if SIM else (1, 4, 9, 12)):
        rc, d_dst, ro, rl = _write(L, M, d_src, offs, lens, hc=level)
        assert rc == int(rl.sum()), (level, rc)
        out = M.down(d_dst)
        for k, d in enumerate(datas):
            rec = out[int(ro[k]):int(ro[k] + rl[k])].tobytes()
            assert int.from_bytes(rec[:4], "little") == len(d) and len(rec) <= _bound(len(d)), (level, k)
            assert port.decompress_safe(rec[4:], len(d)) == (len(d), d), (level, k)
            s, cap = _aligned(d, 7), _bound(len(d))
            host = np.zeros(cap, dtype=np.uint8)
            r = L.b200lz4_compress_HC(s.ctypes.data if len(d) else None, host.ctypes.data, len(d), cap, level)
            assert r > 0 and port.decompress_safe(host[:r].tobytes(), len(d)) == (len(d), d), (level, k)


def _faulty_records(port, rng, n):
    """(blob, cap) pairs: valid records, truncations, flipped bytes, declared lengths off by one either way, negative
    declared lengths, declared lengths larger than the room, records of 0 to 3 bytes"""
    base = port.datagen(1 << 18, 0.5, 0.0, 21).tobytes()
    out = []
    for _ in range(n):
        m = rng.choice((0, 1, 5, 40, 700, 5000) if SIM else (0, 1, 5, 40, 700, 5000, 70000))
        o = rng.randrange(0, 100000)
        data = base[o:o + m] if rng.random() < 0.7 else rng.randbytes(m)
        blob = bytearray(port.with_length_compress(data))
        cap = m
        kind = rng.randrange(9)
        if kind == 1 and len(blob) > 4:
            del blob[rng.randrange(4, len(blob)):]                                  # truncated
        elif kind == 2 and len(blob) > 4:
            for _ in range(rng.randrange(1, 4)):
                i = rng.randrange(4, len(blob)); blob[i] ^= 1 << rng.randrange(8)   # flipped bytes
        elif kind == 3:
            blob[:4] = max(m + rng.choice((-1, 1)), 0).to_bytes(4, "little")        # declared off by one
            cap = m + 1
        elif kind == 4:
            blob[:4] = (0x80000000 | rng.randrange(1 << 20)).to_bytes(4, "little")  # negative declared length
        elif kind == 5:
            cap = max(m - rng.randrange(1, 10), 0)                                  # no room
        elif kind == 6:
            blob = blob[:rng.randrange(0, 4)]                                       # 0 to 3 bytes
        elif kind == 7:
            blob += rng.randbytes(rng.randrange(1, 9))                              # trailing bytes
            cap = m + rng.choice((0, 8))
        out.append((bytes(blob), cap))
    return out


def _read_all(L, M, cases, safe, caps=None):
    """every case in ONE device call, dst ranges with guard bytes between them -> (results, orig_len, dst, doff)"""
    blobs = [b for b, _ in cases]
    caps = [c for _, c in cases] if caps is None else caps
    src, offs, lens = _lay_out(blobs, align=16, phase=3, gap=5)
    doff, pos = [], 7
    for c in caps:
        doff.append(pos)
        pos += int(c) + 24
    d_src, d_dst = M.up(src), M.full(pos + 64, END_GUARD)
    rc, res, orig = _read(L, M, d_src, offs, lens, d_dst, _u64(doff), _u64(caps), safe)
    assert rc == 0, rc
    return res, orig, M.down(d_dst), doff


def test_reader_parity_and_guard_bytes(b200, port):
    """hundreds of valid and faulty records in one call, for both flavours: every result is the host call's, orig_len is the
    declared length (-1 below 4 bytes), the decoded bytes are the host call's, and the writes keep to the rules: nothing
    outside a record's range, nothing at all for a record its header rejects, and on success nothing past the declared length
    (fast) or the result (safe).  A record refused for want of room decodes when read again with dst_cap = orig_len."""
    L, M = b200._native.lib(), _DevMem()
    cases = _faulty_records(port, random.Random(2024), 60 if SIM else 800)
    for safe in (False, True):
        seen = set()
        res, orig, dst, doff = _read_all(L, M, cases, safe)
        for k, (blob, cap) in enumerate(cases):
            want, got_host = _host_read(L, blob, cap, safe)
            declared = int.from_bytes(blob[:4], "little", signed=True) if len(blob) >= 4 else -1
            assert int(res[k]) == want and int(orig[k]) == declared, (safe, k, int(res[k]), want, int(orig[k]), declared)
            got = dst[doff[k]:doff[k] + cap]
            assert (dst[doff[k] + cap:doff[k] + cap + 24] == END_GUARD).all(), (safe, k)
            if len(blob) < 4 or declared < 0 or declared > cap:
                assert want == -1 and (got == END_GUARD).all(), (safe, k)
                seen.add("header")
            elif want >= 0:
                end = want if safe else declared
                assert got[:end].tobytes() == got_host and (got[end:] == END_GUARD).all(), (safe, k)
                seen.add("ok")
            else:
                seen.add("decode")
        assert (dst[:doff[0]] == END_GUARD).all()
        assert seen == {"header", "ok", "decode"}, seen
        again = [k for k, (blob, cap) in enumerate(cases) if int(orig[k]) > cap]
        res2, _, _, _ = _read_all(L, M, [cases[k] for k in again], safe, caps=[int(orig[k]) for k in again])
        assert len(again) > 0 and [int(r) for r in res2] == [_host_read(L, cases[k][0], int(orig[k]), safe)[0] for k in again]
        assert (res2 >= 0).any(), safe
    # the valid records decode to their sources with either flavour
    assert b200.decompress_with_length(port.with_length_compress(b"abc" * 100), safe=True) == b"abc" * 100


def test_round_trip_with_the_writer(b200, port):
    """compress_with_length_dev -> decompress_with_length_dev over many records, both flavours: the sources come back, the
    fast flavour reads each whole record, the safe one decodes each source length"""
    L, M = b200._native.lib(), _DevMem()
    rng = random.Random(5)
    rdg = port.datagen(200000, 0.5, 0.0, 5).tobytes()
    sizes = (0, 1, 100, 4096, 65536, 65537) if SIM else (0, 1, 100, 4096, 65536, 65537, 200000)
    datas = [rdg[:rng.choice(sizes)] for _ in range(24 if SIM else 400)]
    src, offs, lens = _lay_out(datas, align=16, phase=5)
    rc, d_recs, ro, rl = _write(L, M, M.up(src), offs, lens)
    assert rc > 0
    total = int(lens.sum())
    doff = _u64(np.cumsum(lens) - lens)
    for safe in (False, True):
        d_dst = M.full(total + 64, END_GUARD)
        r, res, orig = _read(L, M, d_recs, ro, rl, d_dst, doff, lens, safe)
        out = M.down(d_dst)
        assert r == 0 and (orig == lens.astype(np.int64)).all(), safe
        assert (res == (lens if safe else rl).astype(np.int64)).all(), safe
        assert out[:total].tobytes() == b"".join(datas) and (out[total:] == END_GUARD).all(), safe


def test_errors_launch_nothing_and_write_nothing(b200, port):
    """writer: dst_capacity one short of the bounds (-9), a record of 0x7E000001 bytes, NULL source or destination
    (B200LZ4_E_ARG), no records (0); reader: a NULL result array, NULL offsets, a record of 2^31 bytes, a destination range
    that overflows (B200LZ4_E_ARG; the record declares length 0, so nothing would be written), no records (0): no launch, no
    byte written"""
    L, M = b200._native.lib(), _DevMem()
    datas = [port.datagen(100000, 0.5, 0.0, 6).tobytes(), b"xyz"]
    src, offs, lens = _lay_out(datas)
    d_src = M.up(src)
    cap = sum(_bound(int(n)) for n in lens)
    d_dst = M.full(cap + 64, END_GUARD)
    before = L.b200lz4_launch_count()
    assert _write(L, M, d_src, offs, lens, d_dst=d_dst, cap=cap - 1)[0] == -9
    assert _write(L, M, d_src, offs, _u64([0x7E000001, 3]), d_dst=d_dst, cap=1 << 40)[0] == E_ARG
    ro = np.zeros(2, dtype=np.uint64)
    assert L.b200lz4_compress_with_length_dev(None, offs.ctypes.data, lens.ctypes.data, 2, M.ptr(d_dst), cap, ro.ctypes.data,
                                              ro.ctypes.data, 0, None) == E_ARG
    assert L.b200lz4_compress_with_length_dev(M.ptr(d_src), offs.ctypes.data, lens.ctypes.data, 2, None, cap, None, None, 0,
                                              None) == E_ARG
    assert _write(L, M, d_src, offs[:0], lens[:0], d_dst=d_dst, cap=cap)[0] == 0
    doff, dcap = _u64([0, 100000]), _u64([100000, 3])
    assert _read(L, M, d_src, offs, lens, d_dst, doff, dcap, False, result=False)[0] == E_ARG
    res = np.zeros(2, dtype=np.int64)
    assert L.b200lz4_decompress_with_length_dev(M.ptr(d_src), None, lens.ctypes.data, 2, M.ptr(d_dst), doff.ctypes.data,
                                                dcap.ctypes.data, 1, res.ctypes.data, None, None) == E_ARG
    assert _read(L, M, d_src, offs, _u64([1 << 31, 3]), d_dst, doff, dcap, True)[0] == E_ARG
    d_empty = M.up(np.zeros(5, dtype=np.uint8))                   # length 0, then the empty block's one token
    assert _read(L, M, d_empty, _u64([0]), _u64([5]), d_dst, _u64([2**64 - 2]), _u64([16]), False)[0] == E_ARG
    assert _read(L, M, d_src, offs[:0], lens[:0], d_dst, doff[:0], dcap[:0], True)[0] == 0
    assert L.b200lz4_launch_count() == before
    assert (M.down(d_dst) == END_GUARD).all()


def _expected_writer_launches(lens):
    """per chunk (the writer's rule: at most CHUNK_SPAN source bytes, a longer record alone): one fast-compressor launch per
    size class present (up to 64 KiB, longer), sizes, scan and emit"""
    chunks, cur, span = [], [], 0
    for n in lens:
        if cur and span + n > CHUNK_SPAN:
            chunks.append(cur); cur, span = [], 0
        cur.append(n); span += n
    chunks.append(cur)
    return sum(3 + any(n <= 65536 for n in c) + any(n > 65536 for n in c) for c in chunks)


def test_launch_counts(b200, port):
    """the writer's launches depend on its chunks and their size classes, not on its records: the same bytes as few or many
    records of one class, records of both classes alternating, and calls of several chunks; the reader takes 3 launches for
    1 record and for many"""
    L, M = b200._native.lib(), _DevMem()
    data = port.datagen(1 << 20, 0.5, 0.0, 7).tobytes()
    few, many = (16, 64) if SIM else (16, 4096)
    cases = [[len(data) // few] * few, [len(data) // many] * many,
             [100, 70000] * (4 if SIM else 2048),
             [70000] * (16 if SIM else 4000) + [1000] * 16]                            # more than one chunk
    for lens in cases:
        src = np.frombuffer((data * (sum(lens) // len(data) + 1))[:sum(lens)] + bytes(64), dtype=np.uint8)
        offs = _u64(np.cumsum(lens) - lens)
        before = L.b200lz4_launch_count()
        rc, d_recs, ro, rl = _write(L, M, M.up(src), offs, _u64(lens))
        assert rc > 0 and L.b200lz4_launch_count() - before == _expected_writer_launches(lens), (len(lens), lens[:2])
    assert _expected_writer_launches(cases[0]) == _expected_writer_launches(cases[1]) == 4
    assert _expected_writer_launches(cases[2]) == 5 and _expected_writer_launches(cases[3]) > 5
    for n in (1, 64 if SIM else 4096):
        datas = [data[k * 200:k * 200 + 200] for k in range(n)]
        src, offs, lens = _lay_out(datas, align=16)
        rc, d_recs, ro, rl = _write(L, M, M.up(src), offs, lens)
        d_dst = M.full(200 * n + 64, END_GUARD)
        before = L.b200lz4_launch_count()
        r, res, _ = _read(L, M, d_recs, ro, rl, d_dst, _u64(np.arange(n) * 200), lens, False)
        assert r == 0 and (res == rl.astype(np.int64)).all() and L.b200lz4_launch_count() - before == 3, n


@pytest.mark.skipif(not SIM, reason="the counting emulator build counts the library's host<->device copies")
def test_no_payload_crosses_to_the_host(b200, port):
    """two calls with the same number of records whose payloads differ 64x in size: the writer and both readers copy the same
    bytes between host and device for both, a small constant per record (on the counting emulator library,
    tests/simt/copy_count.h, which test_with_length_sim.py builds)"""
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
    counts = {"write": [], "fast": [], "safe": []}
    for size in (1000, 64000):                                                 # both sizes go to the wide compressor
        datas = [rng.randbytes(size) for _ in range(8)]
        src, offs, lens = _lay_out(datas)
        d_src = M.up(src)
        got = {}
        counts["write"].append(copied(lambda: got.update(w=_write(L, M, d_src, offs, lens))))
        rc, d_recs, ro, rl = got["w"]
        d_dst = M.full(int(lens.sum()) + 64, 0)
        doff = _u64(np.cumsum(lens) - lens)
        for safe in (False, True):
            counts["safe" if safe else "fast"].append(copied(lambda: got.update(r=_read(L, M, d_recs, ro, rl, d_dst, doff, lens, safe))))
            assert got["r"][0] == 0 and (got["r"][1] == (size if safe else rl.astype(np.int64))).all()
    for fn, c in counts.items():
        assert c[0] == c[1], (fn, c)
        assert 0 < c[0][0] and 0 < c[0][1] and sum(c[0]) < 8 * 1000, (fn, c)


@pytest.mark.skipif(SIM, reason="torch streams: GPU only")
def test_ordered_after_a_side_stream(b200, port):
    """the sources are written by torch ops on a side stream and both calls are made on that stream without a synchronise:
    the records hold the new bytes and decode to them"""
    import torch
    old, new = port.datagen(4 << 20, 0.5, 0.0, 1), port.datagen(4 << 20, 0.5, 0.0, 2)
    offs, lens = _u64([0, 3 << 20, (3 << 20) + 65536]), _u64([3 << 20, 65536, (1 << 20) - 65536])
    d_src, d_new = torch.from_numpy(old.copy()).cuda(), torch.from_numpy(new.copy()).cuda()
    d_out = torch.zeros(4 << 20, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.cuda._sleep(20_000_000)                                       # the copy lands well after the call is made
        d_src.copy_(d_new)
        recs, ro, rl = b200.compress_with_length_dev(d_src, offs, lens)
        copy = torch.zeros_like(recs)
        torch.cuda._sleep(20_000_000)
        copy.copy_(recs)                                                    # the reader's input lands well after the call too
        res, orig = b200.decompress_with_length_dev(copy, ro, rl, d_out, offs, lens, safe=True)
    torch.cuda.synchronize()
    host = recs.cpu().numpy()
    L = b200._native.lib()
    for k in range(3):
        rec = host[int(ro[k]):int(ro[k] + rl[k])].tobytes()
        assert rec == _host_record(L, new[int(offs[k]):int(offs[k] + lens[k])].tobytes(), 0), k
    assert (res == lens.astype(np.int64)).all() and (orig == lens.astype(np.int64)).all()
    assert d_out.cpu().numpy().tobytes() == new.tobytes()


@pytest.mark.skipif(SIM, reason="torch tensors: GPU only")
def test_python_wrappers(b200, port):
    import torch
    datas = [port.datagen(300000, 0.5, 0.0, 9).tobytes(), b"", b"abc"]
    src, offs, lens = _lay_out(datas)
    d_src = torch.from_numpy(src).cuda()
    recs, ro, rl = b200.compress_with_length_dev(d_src, list(offs), list(lens))
    assert recs.is_cuda and ro.dtype == np.uint64 and rl.dtype == np.uint64
    host = recs.cpu().numpy()
    for k, d in enumerate(datas):
        rec = host[int(ro[k]):int(ro[k] + rl[k])].tobytes()
        assert rec == b200.compress_with_length(_aligned(d)), k
        assert b200.decompress_with_length(rec) == d and b200.decompress_with_length(rec, safe=True) == d, k
    bound = sum(_bound(int(n)) for n in lens)
    w = torch.full((bound + 100,), END_GUARD, dtype=torch.uint8, device="cuda")
    got, _, _ = b200.compress_with_length_dev(d_src, offs, lens, hc_level=9, out=w)
    assert got.data_ptr() == w.data_ptr() and (w[got.numel():] == END_GUARD).all()
    out = torch.full((400000,), END_GUARD, dtype=torch.uint8, device="cuda")
    doff = [0, 300000, 300100]
    for safe in (False, True):
        res, orig = b200.decompress_with_length_dev(recs, ro, rl, out, doff, [300000, 10, 2], safe=safe)
        assert res.dtype == np.int64 and orig.tolist() == [300000, 0, 3]
        assert res.tolist() == ([300000, 0, -1] if safe else [int(rl[0]), int(rl[1]), -1]), safe
        assert out[:300000].cpu().numpy().tobytes() == datas[0]
    with pytest.raises(ValueError):
        b200.compress_with_length_dev(d_src.cpu(), offs, lens)
    with pytest.raises(ValueError):
        b200.compress_with_length_dev(d_src, offs, [len(src) + 1, 0, 0])
    with pytest.raises(b200.LZ4FrameError) as e:
        b200.compress_with_length_dev(d_src, offs, lens, out=torch.empty(10, dtype=torch.uint8, device="cuda"))
    assert e.value.code == -9
    with pytest.raises(ValueError):
        b200.decompress_with_length_dev(recs, ro, rl, out.cpu(), doff, [1, 1, 1])
    with pytest.raises(ValueError):
        b200.decompress_with_length_dev(recs, ro, rl, out, doff, [1, 1])
    with pytest.raises(ValueError):
        b200.decompress_with_length_dev(recs, ro, rl, out, doff, [1, 1, 400000])
    with pytest.raises(b200.LZ4Exception):
        b200.decompress_with_length(b"\x05\x00\x00\x00\x50abcd" + b"\x00" * 4, safe=True)   # a block that runs past its record
