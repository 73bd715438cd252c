"""CPU count of the fast compressor's verify loads on the bench corpus (RDG P=0.50, seed 2, first 4 blocks of 64 KiB).

Models warp L of lz4_compress_wide_kernel<13>: sub-rounds of 128 positions, lane l holding positions 4l..4l+3, every position
probed and then inserted (same-slot stores: the highest lane and position win, as on the CPU emulator).  Counts how many
candidates are plausible (cand < p), how many share the position's first 4 bytes, and the distinct 128-byte lines the warp's
verify load instructions touch: the parent kernel's two 8-byte loads per candidate, and one 16-byte load (plus one more when
the 8 bytes straddle it) with TAG_BITS-bit hash tags.  Source 16-byte aligned.
    python tools/study/verify_traffic.py"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from oracle import oracle as O  # noqa: E402

HASH_LOG, BS, NBLK = 13, 65536, 4


def lines(addr, on):
    """distinct 128-byte lines per load instruction: addr[sub-round, j, lane], on = the lane issues it"""
    n = 0
    for a, o in zip(addr.reshape(-1, 32), on.reshape(-1, 32)):
        n += len(np.unique(a[o] >> 7))
    return n


def block_counts(d):
    n = len(d)
    mflimit = n - 12
    seq = d[:n - 3].astype(np.uint32) | d[1:n - 2].astype(np.uint32) << 8 | d[2:n - 1].astype(np.uint32) << 16 | d[3:].astype(np.uint32) << 24
    prod = (seq * np.uint32(2654435761)).astype(np.uint32)
    h = prod >> np.uint32(32 - HASH_LOG)
    table = np.zeros(1 << HASH_LOG, dtype=np.int64)
    npos = (mflimit + 1 + 127) // 128 * 128
    cand = np.zeros(npos, dtype=np.int64)
    for s in range(0, npos, 128):
        p = np.arange(s, min(s + 128, mflimit + 1))
        cand[p] = table[h[p]]
        table[h[p]] = p                                  # numpy fancy assignment: the last (highest) position wins
    p = np.arange(npos)
    valid = p <= mflimit
    plaus = valid & (cand < p)
    pv = np.minimum(p, mflimit)
    agree4 = plaus & (seq[cand[pv]] == seq[pv])
    # instruction layout [sub-round, j, lane]: position = 128 * sub-round + 4 * lane + j
    order = lambda x: x.reshape(-1, 32, 4).transpose(0, 2, 1)
    c = cand.copy(); c[~plaus] = 0                       # the parent kernel loads position 0 for implausible candidates
    old = lines(order(c & ~7), order(valid)) + lines(order((c & ~7) + 8), order(valid))
    out = {"positions": int(valid.sum()), "plausible": int(plaus.sum()), "agree4": int(agree4.sum()), "lines_old": old}
    for tb in (0, 1, 2, 4, 8):
        tag = (prod >> np.uint32(32 - HASH_LOG - tb)) & np.uint32((1 << tb) - 1)
        on = plaus & (tag[cand[pv]] == tag[pv])          # a stored position's tag is the tag of its own bytes
        straddle = on & ((cand & 15) > 8)
        out[f"lines_t{tb}"] = lines(order(cand & ~15), order(on)) + lines(order((cand & ~15) + 16), order(straddle))
        out[f"loads_t{tb}"] = int(on.sum())
    return out


def main():
    d = O.best_available().datagen(NBLK * BS, 0.5, 0.0, 2)
    tot = {}
    for b in range(NBLK):
        for k, v in block_counts(d[b * BS:(b + 1) * BS]).items():
            tot[k] = tot.get(k, 0) + v
    print(f"{NBLK} blocks: {tot['positions']} positions, {tot['plausible']} plausible candidates "
          f"({100 * tot['plausible'] / tot['positions']:.1f} %), {100 * tot['agree4'] / tot['plausible']:.1f} % of them agree in 4 bytes")
    print(f"parent kernel (two 8-byte loads): {tot['lines_old'] / NBLK:,.0f} line lookups per block")
    for tb in (0, 1, 2, 4, 8):
        print(f"TAG_BITS={tb}: candidates loaded {100 * tot[f'loads_t{tb}'] / tot['plausible']:5.1f} %, "
              f"line lookups per block {tot[f'lines_t{tb}'] / NBLK:9,.0f} ({100 * tot[f'lines_t{tb}'] / tot['lines_old']:.0f} % of the parent's)")


if __name__ == "__main__":
    main()
