"""The CPU emulator twin of test_block_edges_dev.py: the same hand-built streams and compressor inputs, run through the
kernels' own source on tests/simt (both decoder instantiations, batched and sequential), with dst at every 16-byte
phase between sentinels.  What a decoder must return comes from the CPU checker, never from the stream writer.

Every emulated CTA costs milliseconds, so by default this runs an even slice of each menu (about two minutes);
B200LZ4_EDGES_FULL=1 runs the whole grid, every input length and every phase."""
import os

import numpy as np
import pytest

import lz4_seq as S
from test_kernel_logic_cpu import COMPRESS_KINDS, PAD, csim, msim, sim  # noqa: F401  (module fixtures)

FULL = os.environ.get("B200LZ4_EDGES_FULL") == "1"
SENT = 0xA5


def _buf(b, phase):
    a = np.full(len(b) + 2 * PAD, 0x3C, dtype=np.uint8)
    a[PAD + phase:PAD + phase + len(b)] = np.frombuffer(b, dtype=np.uint8)
    return a, a.ctypes.data + PAD + phase


def _run(fn, src, src_phase, n_src, cap, dst_phase, *extra):
    """one kernel call with the source and dst at the given phases; every byte outside [dst, dst + cap) is a sentinel
    that must come back intact -> (result, dst bytes)"""
    s, sp = _buf(src, src_phase)
    d = np.full(max(cap, 0) + 2 * PAD, SENT, dtype=np.uint8)
    r = fn(sp, n_src, d.ctypes.data + PAD + dst_phase, cap, *extra)
    lo, hi = PAD + dst_phase, PAD + dst_phase + max(cap, 0)
    assert (d[:lo] == SENT).all() and (d[hi:] == SENT).all(), ("wrote outside [dst, dst+cap)", dst_phase, cap)
    return r, d[lo:hi].tobytes()


def _every(items, k):
    return items if FULL else items[::k]


# ------------------------------------------------------------------------------------------------ decoders
CAPS = lambda n: (n, n + 1, n + 5, n + 12, n + 64)


def _check_safe(sim, checker, c, sl, cap, batched, phase, label):
    wr, wo = checker.decompress_safe(c[:sl], cap)
    r, o = _run(sim.sim_decompress_safe, c, phase % 7, sl, cap, phase, batched)
    assert r == wr, (label, "src_len", sl, "cap", cap, "got", r, "want", wr)
    if wr > 0:
        assert o[:wr] == wo, (label, sl, cap)


def _check_fast(sim, checker, c, dl, avail, batched, phase, label):
    pad = c + bytes(dl + dl // 255 + 64)
    avail = min(avail, len(pad))
    wr, wo = checker.decompress_fast(pad, dl)
    if not 0 <= wr <= avail:
        wr = -1                                  # reads past avail: the kernel's one documented deviation
    r, o = _run(sim.sim_decompress_fast, pad, (phase * 3) % 16, avail, dl, phase, batched)
    assert r == wr, (label, "dst_len", dl, "avail", avail, "got", r, "want", wr)
    if wr >= 0:
        assert o == wo, (label, dl, avail)


@pytest.mark.parametrize("batched", [1, 0], ids=["batched", "sequential"])
def test_decoders_end_of_block_grid(sim, checker, batched):
    """a slice of the grid (every case when B200LZ4_EDGES_FULL=1): each case at one of the capacities n, n+1, n+5, n+12,
    n+64 in turn and with the source cut by 1 byte, dst at a phase that moves with the case"""
    grid = S.grid_cases(prefixes=("p20", "p70", "p700", "far") if FULL else ("p20", "p70", "p700"))
    for k, (name, c, n) in enumerate(_every(grid, 13)):
        caps = CAPS(n) if FULL else (CAPS(n)[k % 5],)
        ph = k % 16
        for cap in caps:
            _check_safe(sim, checker, c, len(c), cap, batched, ph, name)
            _check_fast(sim, checker, c, cap, 1 << 30, batched, ph, name)
        for cut in ((1, 2) if FULL else (1 + k % 2,)):
            _check_safe(sim, checker, c, len(c) - cut, n, batched, ph, name)
            _check_fast(sim, checker, c, n, len(c) - cut, batched, ph, name)


@pytest.mark.parametrize("batched", [1, 0], ids=["batched", "sequential"])
def test_decoders_capacity_sweeps(sim, checker, batched):
    """safe: dstCapacity n-80 .. n+150 plus 0, 1, 63, 64, 65; fast: dst_len n-40 .. n+40 on padded input and src_avail
    around the bytes the reference reads"""
    streams = S.random_streams(50, seed=11)
    for k, (name, c, n) in enumerate(_every(streams, 8)):
        ph = (5 * k + 1) % 16
        for cap in sorted(set(range(max(0, n - 80), n + 151)) | {0, 1, 63, 64, 65}):
            _check_safe(sim, checker, c, len(c), cap, batched, ph, name)
        for dl in range(max(0, n - 40), n + 41):
            _check_fast(sim, checker, c, dl, 1 << 30, batched, ph, name)
        r, _ = checker.decompress_fast(c, n)
        read = r if r >= 0 else len(c)
        for a in range(max(0, read - 20), read + 21):
            _check_fast(sim, checker, c, n, a, batched, ph, name)


# ------------------------------------------------------------------------------------------------ compressors
S_HC = [1, 4, 9, 12]                             # one per lazy-depth class of lz4hc_compress_kernel


def _fast_fn(csim, kind):
    return lambda sp, n, dp, cap: csim.sim_compress_fast(sp, n, dp, cap, COMPRESS_KINDS[kind])


def _hc_fn(msim, level):
    return lambda sp, n, dp, cap: msim.sim_compress_hc(sp, n, dp, cap, level, 11, 32)


def _verify(c, d, checker, port, label):
    e = S.strict_check(c, len(d))
    assert e is None, (label, len(d), e)
    assert checker.decompress_safe(c, len(d)) == (len(d), d), label
    jr, jo = port.java_decompress_safe(c, len(d))
    assert jr == len(d) and jo == d, (label, jr)


def test_compressors_at_source_and_dst_phases(csim, msim, checker, port):
    """the <= 64 KiB kernel (three and two warps), the long-block kernel and HC at levels 1 / 4 / 9 / 12, each input at a
    source and a dst phase that move with it (all 16 x 16 when B200LZ4_EDGES_FULL=1), dst_cap = the bound"""
    lengths = list(range(0, 301)) + [65535, 65547, 65548] if FULL else \
        sorted(set(range(0, 301, 11)) | {11, 12, 13, 14, 16, 17, 20, 255, 256, 257})
    fns = [("wide3", _fast_fn(csim, "wide3")), ("wide2", _fast_fn(csim, "wide2")), ("long", _fast_fn(csim, "long"))] + \
          [(f"hc{lv}", _hc_fn(msim, lv)) for lv in S_HC]
    for k, (name, d) in enumerate(S.compress_inputs(lengths)):
        bound = port.compress_bound(len(d))
        chosen = fns if FULL else [fns[k % 3], fns[3 + k % len(S_HC)]]
        for kind, fn in chosen:
            if kind.startswith("wide") and len(d) > 65536:
                continue
            for sp in (range(16) if FULL else (k % 16,)):
                r, c = _run(fn, d, sp, len(d), bound, (7 * sp + k) % 16)
                assert r > 0, (kind, name, sp)
                _verify(c[:r], d, checker, port, (kind, name, sp))


def test_compressors_with_limited_output(csim, msim, checker, port):
    """every capacity from 0 to full + 2: 0 or the full-capacity stream byte for byte (the kernels never shorten the parse
    to fit), never 0 once it fits, and nothing written outside [dst, dst + cap)"""
    lengths = range(0, 301, 7) if FULL else (0, 12, 13, 25, 60)
    for k, (name, d) in enumerate(S.compress_inputs(lengths)):
        if not FULL and k % 2:
            continue
        bound = port.compress_bound(len(d))
        for kind, fn in (("wide3", _fast_fn(csim, "wide3")), ("long", _fast_fn(csim, "long")), ("hc9", _hc_fn(msim, 9))):
            full_r, full = _run(fn, d, 0, len(d), bound, 0)
            assert full_r > 0, (kind, name)
            full = full[:full_r]
            for cap in range(0, full_r + 3):
                r, c = _run(fn, d, cap % 16, len(d), cap, (cap * 5) % 16)
                assert 0 <= r <= cap, (kind, name, cap, r)
                assert r > 0 or cap < full_r, ("fits but refused", kind, name, cap)
                assert r == 0 or c[:r] == full, ("a limited stream differs from the full one", kind, name, cap)
