"""The block decoders and compressors at every end-of-block threshold, byte phase and tight packing.

Decoders: streams built sequence by sequence (tests/lz4_seq.py) put the last match at every distance from the end of the
block, with every final literal run, offsets that take the overlap paths, and prefixes long enough for the batched
decoder's window; capacities sweep every threshold of the safe decoder and both limits of the fast one.  What each call
must return comes from the CPU checker (the reference's own C when it was built, else the pinned port).
Compressors: every source phase, tight destination slots, the u16/u32 table cut-over and limited output.
XXH: the batch kernel's TMA and direct-load paths with per-lane lengths around its chunk boundaries.

Placement: the destination ranges of a batch lie back to back with no gap, the first at each phase 0-15 in turn, and the
sources are unaligned.  Every batch is run as two calls, even-indexed blocks first while the odd ranges hold a
sentinel, then the odd ones: nothing outside a block's own [dst, dst + cap) may change, on success or on error.  Only
the *_batch_dev runs can see a kernel write out of range (there the whole sentinel buffer is the kernel's dst); the
host-buffer pipeline stages dst on the device and copies back only the blocks' own ranges, so its runs check that
pipeline and the results.  Every decoder and compressor test therefore runs through both."""
import random

import numpy as np
import pytest

import lz4_seq as S

pytestmark = pytest.mark.gpu

SENT = 0xA5
GUARD = 64


# ------------------------------------------------------------------------------------------------ layout and calls
def _pack_src(items, phases):
    """items at the given 16-byte phases (after a guard), ascending -> (buffer, offsets, lengths)"""
    offs, pos = [], GUARD
    for it, ph in zip(items, phases):
        pos = (pos + 15) // 16 * 16 + ph
        offs.append(pos)
        pos += len(it) + 1
    buf = np.full(pos + GUARD, 0x3C, dtype=np.uint8)
    for it, o in zip(items, offs):
        buf[o:o + len(it)] = np.frombuffer(it, dtype=np.uint8)
    return buf, np.array(offs, dtype=np.uint64), np.array([len(it) for it in items], dtype=np.int32)


def _host(fn):
    """the call through a *_batch_host entry point.  The pipeline never uploads the caller's dst: the kernel writes into
    device staging and only each block's [dst_off, dst_off + cap) comes back, so a kernel write outside its range
    cannot show here (run_halves still checks that the pipeline's copies stay inside the called blocks' ranges)"""
    def call(src, soff, slen, dst, doff, dcap, *extra):
        return np.asarray(fn(src, soff, slen, dst, doff, dcap, *extra)), dst
    return call


def _dev(fn):
    """the same call through a *_batch_dev entry point: torch tensors, on a non-default stream"""
    import torch
    dev = torch.device("cuda", 0)
    st = torch.cuda.Stream(device=dev)

    def call(src, soff, slen, dst, doff, dcap, *extra):
        with torch.cuda.stream(st):
            t = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a).astype(dt)).to(dev)
            d_dst = t(dst, np.uint8)
            res = torch.full((len(soff),), 0x7FFF0000, dtype=torch.int32, device=dev)
            fn(t(src, np.uint8), t(soff, np.int64), t(slen, np.int32), d_dst, t(doff, np.int64), t(dcap, np.int32), res, *extra)
            st.synchronize()
            dst[:] = d_dst.cpu().numpy()
            return res.cpu().numpy(), dst
    return call


def run_halves(call, src_items, src_phases, src_len, caps, dst_phase, *extra):
    """Run a batch as two calls over tightly packed dst ranges (even blocks, then odd ones) and check that every call
    leaves everything outside its own blocks' ranges as it was.  src_len: per block (None = the item's length).
    -> (results, dst buffer, dst offsets)"""
    n = len(src_items)
    src, soff, ilen = _pack_src(src_items, src_phases)
    slen = ilen if src_len is None else np.asarray(src_len, dtype=np.int32)
    caps = np.asarray(caps, dtype=np.int32)
    widths = np.maximum(caps, 0).astype(np.int64)
    base = GUARD + dst_phase
    doff = (base + np.concatenate([[0], np.cumsum(widths)[:-1]])).astype(np.uint64)
    total = base + int(widths.sum()) + GUARD
    owner = np.full(total, -1, dtype=np.int32)
    owner[base:base + int(widths.sum())] = np.repeat(np.arange(n), widths)
    dst = np.full(total, SENT, dtype=np.uint8)
    res = np.zeros(n, dtype=np.int32)
    for half in (0, 1):
        idx = np.arange(half, n, 2)
        if not len(idx):
            continue
        before = dst.copy()
        r, dst = call(src, soff[idx], slen[idx], dst, doff[idx], caps[idx], *extra)
        res[idx] = r
        mine = (owner >= 0) & (owner % 2 == half)
        moved = np.nonzero((dst != before) & ~mine)[0]
        assert not len(moved), f"half {half}: byte {int(moved[0])} outside the called blocks' ranges changed " \
                               f"(owner {int(owner[moved[0]])}, dst phase {dst_phase})"
    return res, dst, doff


def _groups(n, k=16):
    """case indices split into k interleaved groups: group g is laid out from dst phase g"""
    return [list(range(g, n, k)) for g in range(k)]


# ------------------------------------------------------------------------------------------------ decoder cases
def _safe_cases(streams, caps_of, cuts=(1, 2)):
    """(name, stream as the decoder sees it, cap): every cap of caps_of(n), and the stream cut by 1 and 2 bytes at cap n"""
    out = []
    for name, c, n in streams:
        for cap in caps_of(n):
            out.append((name, c, len(c), cap))
        for cut in cuts:
            out.append((name, c, len(c) - cut, n))
    return out


def check_safe(call, checker, cases, label):
    """cases: (name, stream, src_len, cap) -> every result and decoded byte equals the checker's"""
    want = [checker.decompress_safe(c[:sl], cap) for _, c, sl, cap in cases]
    for g in _groups(len(cases)):
        if not g:
            continue
        sub = [cases[i] for i in g]
        res, dst, doff = run_halves(call, [c for _, c, _, _ in sub], [(3 * i + 1) % 16 for i in g], [sl for _, _, sl, _ in sub],
                                    [cap for _, _, _, cap in sub], g[0] % 16)
        for k, i in enumerate(g):
            wr, wo = want[i]
            name, _, sl, cap = cases[i]
            assert res[k] == wr, (label, name, "src_len", sl, "cap", cap, "got", int(res[k]), "want", wr)
            if wr > 0:
                o = int(doff[k])
                assert dst[o:o + wr].tobytes() == wo, (label, name, sl, cap)
    return sum(1 for r, _ in want if r < 0)


def _fast_expect(checker, c, dl, avail):
    """the reference's result for a stream it may read past `avail` of; the kernel reports -1 exactly when the reference
    would read past avail (its one documented deviation)"""
    r, out = checker.decompress_fast(c, dl)
    return (r, out) if 0 <= r <= avail else (-1, b"")


def check_fast(call, checker, cases, label):
    """cases: (name, stream, dst_len, avail) -> results and dst_len decoded bytes equal the checker's.  The stream is
    followed by dst_len + dst_len/255 + 64 zero bytes, so a reference walking on reads only defined bytes."""
    items, want = [], []
    for name, c, dl, avail in cases:
        pad = c + bytes(max(dl, 0) + max(dl, 0) // 255 + 64)
        items.append(pad)
        want.append(_fast_expect(checker, pad, dl, avail))
    for g in _groups(len(cases)):
        if not g:
            continue
        res, dst, doff = run_halves(call, [items[i] for i in g], [(5 * i + 3) % 16 for i in g], [cases[i][3] for i in g],
                                    [cases[i][2] for i in g], g[0] % 16)
        for k, i in enumerate(g):
            wr, wo = want[i]
            name, _, dl, avail = cases[i]
            assert res[k] == wr, (label, name, "dst_len", dl, "avail", avail, "got", int(res[k]), "want", wr)
            if wr >= 0:
                o = int(doff[k])
                assert dst[o:o + dl].tobytes() == wo, (label, name, dl, avail)
    return sum(1 for r, _ in want if r < 0)


GRID_CAPS = lambda n: (n, n + 1, n + 5, n + 12, n + 64)
SWEEP_CAPS = lambda n: sorted(set(range(max(0, n - 80), n + 151)) | {0, 1, 63, 64, 65})


def fast_grid_cases(streams):
    out = []
    for name, c, n in streams:
        out += [(name, c, dl, 1 << 30) for dl in GRID_CAPS(n)]
        out += [(name, c, n, len(c) - cut) for cut in (1, 2)]
    return out


def fast_sweep_cases(checker, streams):
    out = []
    for name, c, n in streams:
        out += [(name, c, dl, 1 << 30) for dl in range(max(0, n - 40), n + 41)]
        r, _ = checker.decompress_fast(c, n)
        read = r if r >= 0 else len(c)
        out += [(name, c, n, a) for a in range(max(0, read - 20), read + 21)]
    return out


def _entry(b200, kind, path):
    B = b200.batch
    fn = {("safe", "host"): B.decompress_safe_batch_host, ("fast", "host"): B.decompress_fast_batch_host,
          ("safe", "dev"): B.decompress_safe_batch_dev, ("fast", "dev"): B.decompress_fast_batch_dev}[(kind, path)]
    return _host(fn) if path == "host" else _dev(fn)


def _clamp_avail(cases):
    """fast cases carry 'whole padded buffer' as 1 << 30: resolve it to the padded length"""
    return [(nm, c, dl, min(a, len(c) + max(dl, 0) + max(dl, 0) // 255 + 64)) for nm, c, dl, a in cases]


@pytest.fixture(scope="module")
def grid():
    return S.grid_cases()


@pytest.mark.parametrize("path", ["host", "dev"])
def test_safe_decoder_end_of_block_grid(b200, checker, grid, path):
    neg = check_safe(_entry(b200, "safe", path), checker, _safe_cases(grid, GRID_CAPS), "safe grid " + path)
    assert neg > 1000                    # final runs under 5 and short capacities are errors: both sides of every rule


@pytest.mark.parametrize("path", ["host", "dev"])
def test_fast_decoder_end_of_block_grid(b200, checker, grid, path):
    neg = check_fast(_entry(b200, "fast", path), checker, _clamp_avail(fast_grid_cases(grid)), "fast grid " + path)
    assert neg > 1000


@pytest.mark.parametrize("path", ["host", "dev"])
def test_safe_decoder_capacity_sweep(b200, checker, path):
    """dstCapacity from n-80 to n+150 plus 0, 1, 63, 64, 65: every threshold of the safe decoder (64 / 32 / 17 / 16 / 12 /
    8 / 5) and decode_batch's 128 / 256 output margins, on 50 multi-sequence streams"""
    streams = S.random_streams(50, seed=11)
    check_safe(_entry(b200, "safe", path), checker, _safe_cases(streams, SWEEP_CAPS, cuts=(1, 2, 3)), "safe sweep " + path)


@pytest.mark.parametrize("path", ["host", "dev"])
def test_fast_decoder_length_and_avail_sweep(b200, checker, path):
    """dst_len from n-40 to n+40 on padded input, and src_avail from (bytes the reference reads) - 20 to that + 20"""
    streams = S.random_streams(50, seed=12)
    check_fast(_entry(b200, "fast", path), checker, _clamp_avail(fast_sweep_cases(checker, streams)), "fast sweep " + path)


def test_one_block_decoders_at_a_dest_offset(b200, checker, grid):
    """LZ4SafeDecompressor / LZ4FastDecompressor with destOff != 0 (and srcOff != 0): a slice of the grid; the bytes of
    dest outside [destOff, destOff + maxDestLen) stay as they were, on success or on LZ4Exception"""
    f = b200.LZ4Factory.b200Instance()
    for k, (name, c, n) in enumerate(grid[::61]):
        cap = GRID_CAPS(n)[k % 5]
        doff, soff = 1 + k % 15, 3 + k % 13
        wr, wo = checker.decompress_safe(c, cap)
        dest = bytearray(b"\x5A" * (doff + cap + 40))
        src = bytes(soff) + c + b"\x01\x00"
        try:
            r = f.safeDecompressor().decompress(src, soff, len(c), dest, doff, cap)
        except b200.LZ4Exception:
            r = -1
        assert (r >= 0) == (wr >= 0) and (wr < 0 or r == wr), (name, cap, r, wr)
        if wr >= 0:
            assert bytes(dest[doff:doff + wr]) == wo, name
        assert dest[:doff] == b"\x5A" * doff and dest[doff + cap:] == b"\x5A" * 40, name
        # fast: destLen = cap, the readable source ends with the padded stream
        pad = c + bytes(cap + cap // 255 + 64)
        wr, wo = _fast_expect(checker, pad, cap, len(pad))
        dest = bytearray(b"\x5A" * (doff + cap + 40))
        try:
            r = f.fastDecompressor().decompress(bytes(soff) + pad, soff, dest, doff, cap)
        except b200.LZ4Exception:
            r = -1
        assert r == wr, (name, cap, r, wr)
        if wr >= 0:
            assert bytes(dest[doff:doff + cap]) == wo, name
        assert dest[:doff] == b"\x5A" * doff and dest[doff + cap:] == b"\x5A" * 40, name


# ------------------------------------------------------------------------------------------------ compressors
SMALL = list(range(0, 301))
NEAR_64K = list(range(65535, 65549))            # the u16 / u32 table cut-over (LZ4_64Klimit = 65547)
NEAR_1M = [(1 << 20) - 3, (1 << 20) + 3]
HC_LEVELS = [1, 4, 9, 12]                       # one per lazy-depth class of lz4hc_compress_kernel


class _Verdicts:
    """strict_check / checker / java-port verdicts, once per distinct stream"""

    def __init__(self, checker, port):
        self.checker, self.port, self.seen = checker, port, set()

    def check(self, c, d, label):
        key = (len(d), hash(c), hash(d))
        if key in self.seen:
            return
        e = S.strict_check(c, len(d))
        assert e is None, (label, len(d), e)
        r, o = self.checker.decompress_safe(c, len(d))
        assert r == len(d) and o == d, (label, len(d), r)
        jr, jo = self.port.java_decompress_safe(c, len(d))
        assert jr == len(d) and jo == d, (label, len(d), jr)
        self.seen.add(key)


def _compress_call(b200, setting, path):
    B = b200.batch
    fn = {("hc", "host"): B.compress_hc_batch_host, ("fast", "host"): B.compress_fast_batch_host,
          ("hc", "dev"): B.compress_hc_batch_dev, ("fast", "dev"): B.compress_fast_batch_dev}[(setting[0], path)]
    return (_host(fn) if path == "host" else _dev(fn)), (setting[1],)      # max_src_len / level


def compress_batch(b200, setting, path, inputs, src_phases, caps, dst_phase):
    call, extra = _compress_call(b200, setting, path)
    res, dst, doff = run_halves(call, inputs, src_phases, None, caps, dst_phase, *extra)
    return [dst[int(o):int(o) + max(int(r), 0)].tobytes() for o, r in zip(doff, res)], res


SETTINGS = [("fast", 65536), ("fast", 0), ("fast", "exact")] + [("hc", lv) for lv in HC_LEVELS]


@pytest.fixture(scope="module")
def compress_inputs():
    return S.compress_inputs(SMALL + NEAR_64K + NEAR_1M)


@pytest.mark.parametrize("path", ["host", "dev"])
@pytest.mark.parametrize("setting", SETTINGS, ids=lambda s: f"{s[0]}-{s[1]}")
def test_compressors_at_every_source_phase_in_tight_slots(b200, checker, port, compress_inputs, setting, path):
    """every input at every source phase 0-15, destinations back to back with dst_cap = the bound; the fast compressor
    with max_src_len = 65536 (<= 64 KiB kernel), 0 (long-block kernel) and = the block length exactly; HC per lazy class"""
    v = _Verdicts(checker, port)
    items = [(nm, d) for nm, d in compress_inputs if setting != ("fast", 65536) or len(d) <= 65536]
    if setting[1] == "exact":
        by_len = {}
        for nm, d in items:
            by_len.setdefault(len(d), []).append(d)
        for n, ds in by_len.items():
            batch = [(d, ph) for d in ds for ph in range(16)]
            # max_src_len 0 means "no limit" (the long-block kernel): the empty blocks are called with a limit of 1
            outs, res = compress_batch(b200, ("fast", max(n, 1)), path, [d for d, _ in batch], [ph for _, ph in batch],
                                       [port.compress_bound(n)] * len(batch), n % 16)
            for (d, ph), c, r in zip(batch, outs, res):
                assert r > 0, (setting, n, ph)
                v.check(c, d, (setting, n, ph))
        return
    for ph in range(16):
        outs, res = compress_batch(b200, setting, path, [d for _, d in items], [ph] * len(items),
                                   [port.compress_bound(len(d)) for _, d in items], (7 * ph + 5) % 16)
        for (nm, d), c, r in zip(items, outs, res):
            assert r > 0, (setting, nm, ph)
            v.check(c, d, (setting, nm, ph))


def _hc_order_free(d, bucket_log=11, ways=32):
    """True when no hash bucket of lz4hc_compress_kernel (2048 x 32 in the library) ever gets more than `ways`
    positions of this block.  The threads of a CTA claim ways with atomicAdd, so once a bucket wraps, which candidates
    it keeps depends on their order and the parse can differ from run to run; below that every bucket holds the same
    set of positions and the search (longest, then nearest) is a function of that set."""
    n = len(d)
    if n < 13:
        return True
    a = np.frombuffer(d, dtype=np.uint8).astype(np.uint32)
    seq = a[:n - 11] | (a[1:n - 10] << 8) | (a[2:n - 9] << 16) | (a[3:n - 8] << 24)          # positions 0 .. n - 12
    h = ((seq.astype(np.uint64) * 2654435761) & 0xFFFFFFFF) >> (32 - bucket_log)
    return int(np.bincount(h.astype(np.int64)).max()) <= ways


@pytest.mark.parametrize("path", ["host", "dev"])
@pytest.mark.parametrize("setting", [("fast", 65536), ("fast", 0), ("hc", 1), ("hc", 9)], ids=lambda s: f"{s[0]}-{s[1]}")
def test_compressors_with_limited_output(b200, checker, port, setting, path):
    """maxDestLen below the bound: every capacity from 0 to full + 2 for blocks up to 300 bytes, about 40 for 64 KiB
    blocks, each block at the same source phase as its full-capacity run.  The result is 0 or the full-capacity stream
    itself, byte for byte (the kernels never shorten the parse to fit), and never 0 once that fits.  For HC this holds
    where its parse is reproducible (_hc_order_free: random and repeated-tail blocks up to 300 bytes); elsewhere HC
    must return 0 or a valid block of at most cap bytes, and the emulator twin pins the rest, its order being fixed"""
    small = S.compress_inputs(list(range(0, 301, 3)) + [299, 300])
    big = [(nm, d) for nm, d in S.compress_inputs([65536]) if nm != "zeros_65536"] + \
          [("mixed_65536", checker.datagen(65536, 0.5, 0.0, 9).tobytes())]
    items = small + big
    fulls, res = compress_batch(b200, setting, path, [d for _, d in items], [k % 16 for k in range(len(items))],
                                [port.compress_bound(len(d)) for _, d in items], 3)
    v = _Verdicts(checker, port)
    exact = [setting[0] == "fast" or _hc_order_free(d) for _, d in items]
    assert sum(exact) > len(items) // 3, sum(exact)
    cases = []
    rng = random.Random(4)
    for k, ((nm, d), full) in enumerate(zip(items, fulls)):
        assert res[k] > 0, (setting, nm)
        v.check(full, d, (setting, nm))
        F = len(full)
        if len(d) <= 300:
            caps = range(0, F + 3)
        else:
            caps = sorted({0, 1, 15, 16, 17, F // 2, F - 1, F, F + 1, F + 2, F - 5, F - 12, F - 13, F - 16, F - 17}
                          | {rng.randrange(F - 300, F) for _ in range(15)} | {rng.randrange(0, F) for _ in range(10)})
        cases += [(k, cap) for cap in caps]
    for g in _groups(len(cases), 4):
        sub = [cases[i] for i in g]
        outs, rr = compress_batch(b200, setting, path, [items[k][1] for k, _ in sub], [k % 16 for k, _ in sub],
                                  [cap for _, cap in sub], g[0] % 16)
        for (k, cap), c, r in zip(sub, outs, rr):
            (nm, d), full = items[k], fulls[k]
            assert 0 <= r <= cap, (setting, nm, cap, int(r))
            if exact[k]:
                assert r > 0 or cap < len(full), ("fits but refused", setting, nm, cap, len(full))
                assert r == 0 or c == full, ("a limited stream differs from the full one", setting, nm, cap)
            elif r > 0:
                v.check(c, d, (setting, nm, cap))


# ------------------------------------------------------------------------------------------------ XXH batch kernel
XXH_LENS = list(range(0, 16)) + [16, 31, 32, 255, 256, 257, 511, 512, 513, 767, 768, 769, 4095, 4096, 4097]
SEEDS = [0, 0x9747B28C, 0xFFFFFFFF]


def _xxh_layout(rng, nlanes_total, misalign_lane_of_warp):
    """per-lane lengths spread over the chunk and two-stage boundaries within every warp; in the warps listed in
    misalign_lane_of_warp (warp -> (lane, shift)) one lane's buffer starts 1-15 bytes off a 16-byte boundary"""
    lens = [XXH_LENS[(i * 7 + i // 32) % len(XXH_LENS)] for i in range(nlanes_total)]
    offs, pos = [], 0
    for i in range(nlanes_total):
        pos = (pos + 15) // 16 * 16
        w, lane = divmod(i, 32)
        if misalign_lane_of_warp.get(w, (None,))[0] == lane:
            pos += misalign_lane_of_warp[w][1]
            lens[i] = 4097                        # at least one whole stripe, or the lane would not count as unaligned
        offs.append(pos)
        pos += lens[i]
    buf = np.frombuffer(rng.randbytes(pos + 64), dtype=np.uint8).copy()
    return buf, np.array(offs, dtype=np.uint64), np.array(lens, dtype=np.int32)


def _xxh_check(checker, buf, off, ln, h32, h64, seed, label):
    for k in range(len(off)):
        b = buf[int(off[k]):int(off[k]) + int(ln[k])]
        assert int(h32[k]) & 0xFFFFFFFF == checker.xxh32(b, seed), (label, k, int(ln[k]), seed)
        assert int(h64[k]) & (2 ** 64 - 1) == checker.xxh64(b, seed * 0x100000001), (label, k, int(ln[k]), seed)


@pytest.mark.parametrize("n", [1, 31, 33, 100, 129, 300])
def test_xxh_batch_kernel_layouts(b200, checker, n):
    """aligned warps (TMA bulk copies) and warps with one lane off by 1-15 bytes (the whole warp takes the direct loads),
    lane lengths across 256-byte chunks and the two-stage ring, n not a multiple of 32 or 128; host and _dev entries"""
    import torch
    rng = random.Random(n)
    mis = {w: ((w * 11) % 32, 1 + w % 15) for w in range(0, (n + 31) // 32, 2)}       # every other warp: one lane off
    buf, off, ln = _xxh_layout(rng, n, mis)
    B = b200.batch
    dev = torch.device("cuda", 0)
    st = torch.cuda.Stream(device=dev)
    for seed in SEEDS:
        h32 = B.xxh32_batch_host(buf, off, ln, seed)
        h64 = B.xxh64_batch_host(buf, off, ln, seed * 0x100000001)
        _xxh_check(checker, buf, off, ln, h32, h64, seed, "host")
        with torch.cuda.stream(st):
            d_buf = torch.from_numpy(buf).to(dev)
            d_off, d_len = torch.from_numpy(off.astype(np.int64)).to(dev), torch.from_numpy(ln).to(dev)
            o32 = torch.zeros(n, dtype=torch.int32, device=dev); o64 = torch.zeros(n, dtype=torch.int64, device=dev)
            B.xxh32_batch_dev(d_buf, d_off, d_len, o32, seed)
            B.xxh64_batch_dev(d_buf, d_off, d_len, o64, seed * 0x100000001)
            st.synchronize()
        _xxh_check(checker, buf, off, ln, o32.cpu().numpy(), o64.cpu().numpy(), seed, "dev")


def test_xxh_host_path_picks_either_kernel(b200, checker):
    """host batches whose average length falls on each side of XXH_LONG_AVG (32 KiB): the per-lane batch kernel and the
    one-warp-per-stream kernel, same layouts and seeds"""
    rng = random.Random(77)
    for long_avg in (False, True):
        n = 70
        lens = [XXH_LENS[i % len(XXH_LENS)] + ((40000, 30000)[i % 2] if long_avg else 0) for i in range(n)]
        offs, pos = [], 0
        for i, L in enumerate(lens):
            pos += (i * 5) % 16
            offs.append(pos); pos += L
        buf = np.frombuffer(rng.randbytes(pos + 64), dtype=np.uint8).copy()
        off, ln = np.array(offs, dtype=np.uint64), np.array(lens, dtype=np.int32)
        assert (sum(lens) / n >= 32768) == long_avg
        for seed in SEEDS:
            _xxh_check(checker, buf, off, ln, b200.batch.xxh32_batch_host(buf, off, ln, seed),
                       b200.batch.xxh64_batch_host(buf, off, ln, seed * 0x100000001), seed, ("long average", long_avg))
