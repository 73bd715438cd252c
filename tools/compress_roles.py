"""Per-role cycle breakdown of the <= 64 KiB fast compressor (lz4_compress_wide_kernel) at the bench shape.

Needs a library built with the trace counters (they are not in the default build):
    tools/build_variants.sh trace:"-DB200_WIDE_TRACE"          # add -DB200_WIDE_TAG_BITS=N for another tag width
    B200LZ4_TEST_SO=variants/libb200lz4_trace.so python tools/compress_roles.py
Every 64th CTA records, per warp, the clock64 cycles it spent in total and in its waits (L at BAR_FREE, P at BAR_FULL and
BAR_REC_FREE, E at BAR_REC_FULL) and P's cycles in extend() and search(); this prints their means over the sampled CTAs.
The counters cost a few instructions of their own, so the traced kernel is a little slower than the product build."""
import ctypes
import os
import sys

import numpy as np
import torch

import _variant  # noqa: F401  (B200LZ4_TEST_SO)
import lz4java_b200 as L
from oracle import oracle as O

NAMES = ["L_total", "L_wait_free", "E_total", "E_wait_rec_full", "P_total", "P_wait_full", "P_wait_rec_free", "P_extend",
         "P_search", "sequences", "extends", "searches"]          # the row layout of g_wide_trace (WT_* in the kernel)
EVERY = 64


def main():
    nblk = int(os.environ.get("NBLK", 524288)); bs = 65536
    lib = L._native.lib()
    if not hasattr(lib, "b200lz4_wide_trace_read"):
        sys.exit("this library has no trace counters: build it with -DB200_WIDE_TRACE (see the docstring)")
    lib.b200lz4_wide_trace_read.restype = ctypes.c_int
    lib.b200lz4_wide_trace_read.argtypes = [ctypes.c_void_p, ctypes.c_int]
    dev = torch.device("cuda:0")
    base_n = min(nblk, 4096)                                     # the bench corpus: RDG P=0.50 seed 2, tiled, blocks made distinct
    base = torch.from_numpy(O.best_available().datagen(base_n * bs, 0.5, 0.0, 2)).to(dev)
    src = base.repeat((nblk + base_n - 1) // base_n)[: nblk * bs].contiguous()
    v = src.view(nblk, bs)
    idx = torch.arange(nblk, device=dev, dtype=torch.int64)
    for k in range(8):
        v[:, k] ^= ((idx >> (8 * k)) & 0xFF).to(torch.uint8)
    bound = L.max_compressed_length(bs); stride = (bound + 15) // 16 * 16
    soff = idx * bs
    slen = torch.full((nblk,), bs, device=dev, dtype=torch.int32)
    coff = idx * stride
    ccap = torch.full((nblk,), bound, device=dev, dtype=torch.int32)
    comp = torch.empty(nblk * stride, device=dev, dtype=torch.uint8)
    clen = torch.zeros(nblk, device=dev, dtype=torch.int32)
    for _ in range(3):                                           # the last launch's counters are read
        L.batch.compress_fast_batch_dev(src, soff, slen, comp, coff, ccap, clen, bs)
    torch.cuda.synchronize()
    rows = (nblk + EVERY - 1) // EVERY
    t = np.zeros((rows, len(NAMES)), dtype=np.uint64)
    if lib.b200lz4_wide_trace_read(t.ctypes.data, rows) != len(NAMES):
        sys.exit("b200lz4_wide_trace_read failed")
    m = t.astype(np.float64).mean(axis=0)
    cyc = dict(zip(NAMES, m))
    total = max(cyc["L_total"], cyc["P_total"], cyc["E_total"])
    print(f"{lib.b200lz4_wide_trace_ctas_per_sm()} CTAs per SM (cudaOccupancyMaxActiveBlocksPerMultiprocessor)")
    print(f"{rows} sampled CTAs of {nblk} x 64 KiB blocks; mean cycles per CTA (share of the longest warp's {total:,.0f})")
    for k in NAMES[:9]:
        print(f"  {k:18s} {cyc[k]:14,.0f}  {100 * cyc[k] / total:5.1f} %")
    seq = cyc["sequences"]
    print(f"  per CTA: {seq:,.0f} sequences, {cyc['extends']:,.0f} extends, {cyc['searches']:,.0f} searches; "
          f"{total / max(seq, 1):.0f} cycles per sequence")
    for who, busy in (("L", cyc["L_total"] - cyc["L_wait_free"]),
                      ("P", cyc["P_total"] - cyc["P_wait_full"] - cyc["P_wait_rec_free"]),
                      ("E", cyc["E_total"] - cyc["E_wait_rec_full"])):
        print(f"  {who} outside its waits: {busy:14,.0f}  {100 * busy / total:5.1f} %")


if __name__ == "__main__":
    main()
