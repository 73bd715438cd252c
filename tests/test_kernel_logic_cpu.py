"""The CUDA kernels' own source, run on the CPU by a SIMT emulator (tests/simt/simt.h), against the oracle.

No GPU is involved and nothing here is a product path: the .cu files of lz4-java_b200/csrc are compiled as host C++
with -DB200_HOST_SIM (every CUDA thread of a CTA becomes a coroutine; warp collectives, __syncthreads and the named
barriers of the two-warp compressor are emulated; a deadlock or a divergent full-mask collective aborts).  The four
decoder kernels — safe/fast x batched/sequential — and the fast-compress kernels (algos 1-3, all table variants) are
fuzzed on inputs the GPU tests also use.  This checks the kernels' logic (token walk, margins, dependency rounds,
the reference's accept/reject rules and return codes, the parser/lookup hand-off), not timing or the GPU memory model.  It exists because the build box has no GPU: a logic bug in the batched decoder
(a long sequence early in a batch pushing later ones past the output margin) was found late in round 1 by a GPU
sweep; on the pre-fix source this file's test_walk_stops_at_the_stream_end fails on the same six blocks a CPU model
predicted, on the fixed source it passes."""
import ctypes
import os
import random
import subprocess

import numpy as np
import pytest

import corpus

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
PAD = 4096


def _build(harness, so_name):
    out = os.path.join(HERE, "simt", "_build")
    os.makedirs(out, exist_ok=True)
    so = os.path.join(out, so_name)
    cmd = ["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-Wno-unknown-pragmas", "-Wno-attributes", "-DB200_HOST_SIM",
           "-I" + os.path.join(HERE, "simt"), "-I" + os.path.join(ROOT, "lz4-java_b200", "csrc"),
           os.path.join(HERE, "simt", harness), "-o", so]
    subprocess.run(cmd, check=True, capture_output=True)
    return ctypes.CDLL(so)


@pytest.fixture(scope="module")
def sim():
    lib = _build("dec_harness.cpp", "libdecsim.so")
    for f in (lib.sim_decompress_safe, lib.sim_decompress_fast):
        f.restype = ctypes.c_int
        f.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_int]
    return lib


@pytest.fixture(scope="module")
def msim():
    lib = _build("misc_harness.cpp", "libmiscsim.so")
    lib.sim_compress_hc.restype = ctypes.c_int
    lib.sim_compress_hc.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int]
    lib.sim_compact.restype = None
    lib.sim_compact.argtypes = [ctypes.c_void_p] * 6 + [ctypes.c_uint32]
    lib.sim_xxh32_long.restype = ctypes.c_uint32; lib.sim_xxh32_long.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_uint32]
    lib.sim_xxh64_long.restype = ctypes.c_uint64; lib.sim_xxh64_long.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_uint64]
    lib.sim_xxh32_stream.restype = ctypes.c_uint32
    lib.sim_xxh32_stream.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_uint32, ctypes.c_void_p, ctypes.c_int]
    lib.sim_xxh64_stream.restype = ctypes.c_uint64
    lib.sim_xxh64_stream.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_uint64, ctypes.c_void_p, ctypes.c_int]
    return lib


@pytest.fixture(scope="module")
def csim():
    lib = _build("comp_harness.cpp", "libcompsim.so")
    lib.sim_compress_fast.restype = ctypes.c_int
    lib.sim_compress_fast.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_int]
    return lib


def _src(b):
    a = np.zeros(len(b) + 2 * PAD, dtype=np.uint8)
    a[PAD:PAD + len(b)] = np.frombuffer(b, dtype=np.uint8)
    return a


def run_safe(sim, c, cap, batched):
    s = _src(c); d = np.full(max(cap, 0) + 2 * PAD, 0x55, dtype=np.uint8)
    r = sim.sim_decompress_safe(s.ctypes.data + PAD, len(c), d.ctypes.data + PAD, cap, batched)
    assert (d[:PAD] == 0x55).all() and (d[PAD + max(cap, 0):] == 0x55).all(), "wrote outside [dst, dst+cap)"
    return r, d[PAD:PAD + max(r, 0)].tobytes()


def run_fast(sim, c, n, batched, readable=None):
    """readable: bytes the decoder may read (>= the stream); default = the stream itself"""
    data = c if readable is None else readable
    s = _src(data); d = np.full(n + 2 * PAD, 0x55, dtype=np.uint8)
    r = sim.sim_decompress_fast(s.ctypes.data + PAD, len(data), d.ctypes.data + PAD, n, batched)
    assert (d[:PAD] == 0x55).all() and (d[PAD + n:] == 0x55).all(), "wrote outside [dst, dst+n)"
    return r, d[PAD:PAD + n].tobytes()


@pytest.mark.parametrize("batched", [1, 0], ids=["batched", "sequential"])
def test_corpus_round_trips(sim, port, batched):
    for name, d in corpus.blocks(port):
        if len(d) > 300000:
            continue
        c = port.compress(d)
        r, o = run_safe(sim, c, len(d), batched)
        assert r == len(d) and o == d, (name, r)
        r, o = run_fast(sim, c, len(d), batched)
        assert r == len(c) and o == d, (name, r)


@pytest.mark.parametrize("batched", [1, 0], ids=["batched", "sequential"])
def test_safe_decoder_return_codes_on_malformed_input(sim, port, batched):
    """same accept/reject set and the same negative codes as the reference (lz4.c:2337), like the GPU test"""
    rng = random.Random(99)
    cases = []
    for name, d in corpus.blocks(port, big=False)[::3]:
        c = port.compress(d); n = len(d)
        for cap in (n, n - 1, n + 1, n + 64, max(0, n - 13), 0, n // 2):
            cases.append((c, cap))
        for cut in (1, 3, 8):
            if len(c) > cut:
                cases.append((c[:-cut], n))
        cases.append((c + b"\x10\x41", n))
        for m in corpus.mutate(c, rng, 6):
            cases.append((m, rng.choice([n, n + 1, n - 1, n + 70])))
    for v in corpus.MALFORMED:
        for cap in (20, 64, 200):
            cases.append((v, cap))
    negatives = 0
    for k, (c, cap) in enumerate(cases):
        if not c:
            continue
        want, out = port.decompress_safe(c, cap)
        r, o = run_safe(sim, c, cap, batched)
        assert r == want, (k, len(c), cap, r, want, c[:16].hex())
        if want >= 0:
            assert o == out, k
        else:
            negatives += 1
    assert negatives > 50


@pytest.mark.parametrize("batched", [1, 0], ids=["batched", "sequential"])
def test_fast_decoder_on_malformed_input(sim, port, batched):
    rng = random.Random(7)
    for name, d in corpus.blocks(port, big=False)[::4]:
        c = port.compress(d); n = len(d)
        cases = [(c, dl) for dl in (n, n - 1, n + 1, n + 5, max(0, n - 12)) if dl >= 0]
        cases += [(m, n) for m in corpus.mutate(c, rng, 4)]
        for cc, dl in cases:
            if not cc:
                continue
            padded = cc + bytes(dl + dl // 255 + 64)          # the reference's unbounded reads stay defined
            want, out = port.decompress_fast(padded, dl)
            r, o = run_fast(sim, padded, dl, batched)
            assert r == want, (name, len(cc), dl, r, want)
            if want >= 0:
                assert o == out, name


def _tail_heavy_blocks():
    rng = random.Random(8080)
    items = []
    for trial in range(96):
        hist = bytes(rng.randrange(256) for _ in range(3000))
        parts = [hist]

        def short():
            parts.append(bytes(rng.randrange(256) for _ in range(rng.randrange(1, 7))))
            a = rng.randrange(0, 2900); parts.append(hist[a:a + rng.randrange(5, 13)])
        for _ in range(rng.randrange(40, 90)): short()
        a = rng.randrange(0, 500)
        parts.append(bytes(rng.randrange(256) for _ in range(2))); parts.append(hist[a:a + rng.randrange(1100, 1700)])
        for _ in range(rng.randrange(3, 26)): short()
        parts.append(bytes(rng.randrange(256) for _ in range(rng.randrange(5, 15))))
        items.append(b"".join(parts))
    return items


@pytest.mark.parametrize("batched", [1, 0], ids=["batched", "sequential"])
def test_walk_stops_at_the_stream_end(sim, port, batched):
    """the data of tests/test_gpu_parity.py::test_decompress_fast_does_not_walk_past_the_stream: what follows each
    stream starts with a valid-looking offset and continues with another block's sequences"""
    items = _tail_heavy_blocks()
    comp = [port.compress(d) for d in items]
    for k, (d, c) in enumerate(zip(items, comp)):
        readable = c + b"\x01\x00" + comp[(k + 1) % len(comp)][9:3000] + bytes(64)
        r, o = run_fast(sim, c, len(d), batched, readable=readable)
        assert r == len(c) and o == d, (k, r, len(c))
        r, o = run_safe(sim, c, len(d) + (k % 3) * 40, batched)
        assert r == len(d) and o == d, (k, r)


@pytest.mark.parametrize("batched", [1, 0], ids=["batched", "sequential"])
def test_dependency_patterns_and_extremes(sim, port, batched):
    rng = random.Random(4242)
    items = [bytes(70000), bytes([7]) * 40000 + bytes(rng.randrange(256) for _ in range(300)) + bytes([9]) * 3000,
             bytes(rng.randrange(256) for _ in range(20000))]
    for trial in range(10):
        parts = []
        while sum(map(len, parts)) < 20000 + 3000 * trial:
            kind = rng.randrange(7)
            if kind == 0:
                parts.append(bytes([rng.randrange(256)]) * rng.randrange(5, 700))
            elif kind == 1:
                pat = bytes(rng.randrange(256) for _ in range(rng.randrange(2, 9))); parts.append(pat * rng.randrange(3, 120))
            elif kind == 2:
                parts.append(bytes(rng.randrange(256) for _ in range(rng.randrange(1, 80))))
            elif kind == 3 and parts:
                prev = b"".join(parts[-3:]); a = rng.randrange(len(prev)); parts.append(prev[a:a + rng.randrange(4, 60)])
            elif kind == 4 and parts:
                whole = b"".join(parts); a = rng.randrange(len(whole)); parts.append(whole[a:a + rng.randrange(4, 400)])
            elif kind == 5:
                pat = bytes(rng.randrange(256) for _ in range(rng.randrange(33, 200))); parts.append(pat * rng.randrange(2, 6))
            else:
                parts.append(bytes(rng.randrange(4) for _ in range(rng.randrange(20, 300))))
        items.append(b"".join(parts))
    for k, d in enumerate(items):
        c = port.compress(d)
        r, o = run_safe(sim, c, len(d), batched)
        assert r == len(d) and o == d, (k, r)
        r, o = run_fast(sim, c, len(d), batched, readable=c + bytes(3000))
        assert r == len(c) and o == d, (k, r)


# ---------------------------------------------------------------------------------------------- fast compress
COMPRESS_KINDS = {"wide3": 3, "wide2": 2, "long": 0}     # <= 64 KiB kernel with three / two warps per block; long-block kernel (32-bit table)


def run_compress(csim, d, cap, kind, shift=0):
    a = np.zeros(len(d) + 2 * PAD + 8, dtype=np.uint8)
    a[PAD + shift:PAD + shift + len(d)] = np.frombuffer(d, dtype=np.uint8)
    o = np.full(max(cap, 0) + 2 * PAD, 0x55, dtype=np.uint8)
    r = csim.sim_compress_fast(a.ctypes.data + PAD + shift, len(d), o.ctypes.data + PAD, cap, COMPRESS_KINDS[kind])
    assert (o[:PAD] == 0x55).all() and (o[PAD + max(cap, 0):] == 0x55).all(), "wrote outside [dst, dst+cap)"
    return r, o[PAD:PAD + max(r, 0)].tobytes()


@pytest.mark.parametrize("kind", list(COMPRESS_KINDS))
def test_compress_kernels_emit_valid_blocks(csim, port, kind):
    tot = ctot = 0
    for name, d in corpus.blocks(port):
        if len(d) > 70000 or (kind != "long" and len(d) >= 65536 + 11):
            continue
        r, c = run_compress(csim, d, port.compress_bound(len(d)), kind)
        assert r > 0, (kind, name)
        rr, o = port.decompress_safe(c, len(d))
        assert rr == len(d) and o == d, (kind, name, len(d), rr)
        tot += len(d); ctot += r
    assert tot / ctot > 1.9                      # the corpus compresses about 2.0-2.35x with every kernel


def test_compress_streams_are_the_pinned_ones(csim, port):
    """tests/golden/fast_streams.json: the <= 64 KiB kernel's bytes on the seeded corpus (both builds, word-aligned source) —
    the same bytes the round-1 kernel emitted, so a refactor that changes the parse shows up here.  Chunks are cut on
    the source's aligned words, so a source that starts 1..3 bytes into a word may parse differently (still valid, and
    the two builds still agree): those alignments are checked for that"""
    import hashlib, json
    gold = json.load(open(os.path.join(HERE, "golden", "fast_streams.json")))["streams"]
    seen = 0
    for name, d in corpus.blocks(port):
        if name not in gold:
            continue
        for kind in ("wide3", "wide2"):
            r, c = run_compress(csim, d, port.compress_bound(len(d)), kind)
            assert (r, hashlib.sha256(c).hexdigest()) == (gold[name]["c"], gold[name]["sha256"]), (name, kind)
        for shift in (1, 3):
            r3, c3 = run_compress(csim, d, port.compress_bound(len(d)), "wide3", shift)
            assert (r3, c3) == run_compress(csim, d, port.compress_bound(len(d)), "wide2", shift), (name, shift)
            assert port.decompress_safe(c3, len(d)) == (len(d), d), (name, shift)
        seen += 1
    assert seen == len(gold)


@pytest.mark.parametrize("kind", list(COMPRESS_KINDS))
def test_compress_limited_output_never_overruns(csim, port, kind):
    """maxDestLen below the bound (lz4.c:1085-1088, 1158, 1269-1279): either a valid block that fits, or 0; a negative
    capacity is "no room" (0 and nothing written), never a wrapped unsigned comparison"""
    rng = random.Random(5)
    picks = [d for _, d in corpus.blocks(port, big=False)][::5]
    for d in picks:
        full, _ = run_compress(csim, d, port.compress_bound(len(d)), kind)
        for cap in sorted({-1, -(1 << 31), 0, 1, full - 1, full, full + 1, max(0, full // 2), max(0, full - 17), rng.randrange(0, full + 20)}):
            r, c = run_compress(csim, d, cap, kind)
            assert 0 <= r <= max(cap, 0)
            if r > 0:
                rr, o = port.decompress_safe(c, len(d))
                assert rr == len(d) and o == d
            elif cap >= full:
                raise AssertionError(("fits but was refused", len(d), cap, full))


# ---------------------------------------------------------------------------------------------- HC, long-stream / streaming XXH
def test_long_stream_and_streaming_xxh_kernels(msim, port):
    """xxh32_long_kernel / xxh64_long_kernel (one warp per stream) and the warp-cooperative streaming updates:
    every alignment phase, lengths around the stripe / row / group boundaries, random chunkings, digest mid-stream"""
    rng = random.Random(3)
    sizes = [0, 1, 3, 4, 15, 16, 17, 31, 32, 33, 63, 64, 127, 128, 129, 255, 256, 257, 1023, 1024, 1025, 4096, 5000, 8191, 8192, 8193, 40000, 70001]
    for trial, n0 in enumerate(sizes * 2):
        n = n0 + (rng.randrange(0, 40) if trial >= len(sizes) else 0)
        ph = trial % 8
        d = rng.randbytes(n)
        a = np.zeros(n + 2 * PAD, dtype=np.uint8); a[PAD + ph:PAD + ph + n] = np.frombuffer(d, dtype=np.uint8)
        ptr = a.ctypes.data + PAD + ph
        for seed in (0, 0x9747B28C):
            assert msim.sim_xxh32_long(ptr, n, seed) == port.xxh32(d, seed), (n, ph, seed)
            assert msim.sim_xxh64_long(ptr, n, seed) == port.xxh64(d, seed), (n, ph, seed)
        cuts = sorted(rng.randrange(0, n + 1) for _ in range(rng.randrange(0, 6)))
        ca = (ctypes.c_int * max(1, len(cuts)))(*cuts)
        assert msim.sim_xxh32_stream(ptr, n, 7, ca, len(cuts)) == port.xxh32(d, 7), (n, cuts)
        assert msim.sim_xxh64_stream(ptr, n, 7, ca, len(cuts)) == port.xxh64(d, 7), (n, cuts)


@pytest.mark.parametrize("table", [(11, 32), (10, 16)], ids=["2048x32", "1024x16"])
def test_hc_kernel_emits_valid_blocks(msim, port, table):
    bl, ways = table
    picks = [(n, d) for n, d in corpus.blocks(port, big=False) if len(d) <= 8192][::2]
    assert len(picks) > 15
    for name, d in picks:
        bound = port.compress_bound(len(d))
        s = _src(d); o = np.full(bound + 2 * PAD, 0x55, dtype=np.uint8)
        r = msim.sim_compress_hc(s.ctypes.data + PAD, len(d), o.ctypes.data + PAD, bound, 9, bl, ways)
        assert r > 0 and (o[:PAD] == 0x55).all() and (o[PAD + bound:] == 0x55).all(), (name, r)
        rr, oo = port.decompress_safe(o[PAD:PAD + r].tobytes(), len(d))
        assert rr == len(d) and oo == d, (name, bl, ways)
        if len(d) >= 2048 and name.startswith(("rdg", "text", "rand3")):
            assert r <= len(port.compress(d)) * 1.02, (name, r)          # never meaningfully worse than the fast parse


def test_compaction_scan_and_gather(msim):
    """compact.cu: exclusive scan of the lengths by one 1024-thread CTA (crossing its 1024-entry rounds), then the gather"""
    rng = random.Random(12)
    for n in (1, 2, 31, 32, 33, 1023, 1024, 1025, 2500):
        lens = np.array([rng.choice([0, -3, 1, 5, 17, 40, 100, 333]) for _ in range(n)], dtype=np.int32)
        stride = 352
        slots = np.frombuffer(rng.randbytes(n * stride), dtype=np.uint8).copy()
        slot_off = (np.arange(n, dtype=np.uint64) * stride)
        out = np.full(int(np.maximum(lens, 0).sum()) + 64, 0x55, dtype=np.uint8)
        out_off = np.zeros(n, dtype=np.uint64); total = np.zeros(1, dtype=np.uint64)
        msim.sim_compact(slots.ctypes.data, slot_off.ctypes.data, lens.ctypes.data, out.ctypes.data, out_off.ctypes.data, total.ctypes.data, n)
        want_off = np.concatenate([[0], np.cumsum(np.maximum(lens, 0))[:-1]]).astype(np.uint64)
        assert (out_off == want_off).all() and int(total[0]) == int(np.maximum(lens, 0).sum()), n
        packed = b"".join(slots[k * stride:k * stride + max(int(lens[k]), 0)].tobytes() for k in range(n))
        assert out[:len(packed)].tobytes() == packed and (out[len(packed):] == 0x55).all(), n


# ---------------------------------------------------------------------------------------------- the host layer too
@pytest.fixture(scope="module")
def sim_library():
    subprocess.run(["bash", os.path.join(HERE, "simt", "build_sim_library.sh")], check=True, capture_output=True)
    return os.path.join(HERE, "simt", "_build", "libb200lz4_sim.so")


def test_host_layer_on_the_emulator_library(sim_library):
    """tests/simt/build_sim_library.sh builds the WHOLE library for the emulator (capi.cu / frame.cu / containers.cu
    unchanged over a stand-in CUDA runtime); a few of the GPU parity tests then run against it in a subprocess (the
    product loader of this process is left alone): the batch pipeline with bounce buffers and compaction, the
    single-block factory API with its exception contract, streaming hashes, the drain of a pipeline call that
    fails half way, the JNI shim, the range-sharded multi-GPU calls and the device-side stitch over three pretend devices (SIMT_DEVICES), frames written with flush().  The full file takes ~20 minutes this way
    (see tests/simt/README.md); this is the one-minute slice."""
    import sys
    # 1 MiB pipeline chunks: the 40-block batches of these tests then cross chunk boundaries (all three stream slots in use)
    env = dict(os.environ, B200LZ4_TEST_SO=sim_library, B200LZ4_CHUNK_MB="1", SIMT_DEVICES="3")
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.join(HERE, "test_gpu_parity.py"), "-m", "gpu", "-q", "-x", "-p", "no:cacheprovider",
                        "-W", "ignore::DeprecationWarning", "-k", "factory_api or compact_host or xxhash_streaming or self_roundtrip or failed_pipeline or contexts_are_reused or jni_shim or multi_gpu_range or written_with_flush or device_side_compaction or stream_order"],
                       env=env, cwd=ROOT, capture_output=True, text=True)
    assert r.returncode == 0 and "11 passed" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]


_FAILED_ALLOC = r"""
import ctypes, os, sys
import numpy as np
lib = ctypes.CDLL(sys.argv[1])
lib.b200xxh64_batch_host.argtypes = [ctypes.c_void_p] * 3 + [ctypes.c_uint64, ctypes.c_void_p, ctypes.c_size_t]
lib.b200lz4_last_error.restype = ctypes.c_char_p
buf = np.random.default_rng(5).integers(0, 256, 100 * 64, dtype=np.uint8)
off, ln = np.arange(100, dtype=np.uint64) * np.uint64(64), np.full(100, 64, dtype=np.int32)
def hash_(n):
    out = np.zeros(n, dtype=np.uint64)
    return lib.b200xxh64_batch_host(buf.ctypes.data, off.ctypes.data, ln.ctypes.data, 0, out.ctypes.data, n), out
rc, first = hash_(10)
assert rc == 0, rc
os.environ["SIMT_FAIL_HOST_ALLOC"] = "1"
rc, _ = hash_(100)                          # the slot's descriptor arrays must grow: the pinned half fails
del os.environ["SIMT_FAIL_HOST_ALLOC"]
assert rc < 0 and b"cudaHostAlloc" in lib.b200lz4_last_error(), (rc, lib.b200lz4_last_error())
rc, again = hash_(10)
assert rc == 0 and (again == first).all(), rc
print("ok")
"""


def test_failed_staging_allocation_leaves_the_slot_usable(sim_library):
    """A pipeline slot whose staging cannot grow (the pinned allocation fails after the old buffer was freed) fails that
    call with a CUDA error, and the next, smaller call on the thread allocates again instead of staging through the
    freed buffer.  Runs in a subprocess: the regression is a crash."""
    import sys
    r = subprocess.run([sys.executable, "-c", _FAILED_ALLOC, sim_library], capture_output=True, text=True)
    assert r.returncode == 0 and r.stdout.strip() == "ok", (r.returncode, r.stdout[-2000:] + r.stderr[-2000:])
