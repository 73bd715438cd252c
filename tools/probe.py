"""Quick device-resident throughput probe (development aid; bench.py is the contract)."""
import sys, os, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
import _variant  # noqa: F401  (B200LZ4_TEST_SO development switch)
import lz4java_b200 as L
from oracle import oracle as O

def timeit(fn, iters=5, warm=2):
    for _ in range(warm): fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record(); torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) / 1e3)
    return min(ts), sorted(ts)[len(ts)//2]

def main():
    nblk = int(os.environ.get("NBLK", 16384)); bs = int(os.environ.get("BS", 65536)); mp = float(os.environ.get("MP", 0.5))
    chk = O.best_available()
    base_n = min(nblk, 4096)
    host = chk.datagen(base_n * bs, mp, 0.0, 2)
    dev = torch.device("cuda:0")
    base = torch.from_numpy(host).to(dev)
    reps = (nblk + base_n - 1) // base_n
    src = base.repeat(reps)[: nblk * bs].contiguous()
    # perturb first 8 bytes of each block so blocks are distinct
    v = src.view(nblk, bs)
    idx = torch.arange(nblk, device=dev, dtype=torch.int64)
    for k in range(4):
        v[:, k] = v[:, k] ^ ((idx >> (8 * k)) & 0xFF).to(torch.uint8)
    bound = L.max_compressed_length(bs); stride = (bound + 15) // 16 * 16
    soff = (torch.arange(nblk, device=dev, dtype=torch.int64) * bs)
    slen = torch.full((nblk,), bs, device=dev, dtype=torch.int32)
    coff = (torch.arange(nblk, device=dev, dtype=torch.int64) * stride)
    ccap = torch.full((nblk,), bound, device=dev, dtype=torch.int32)
    comp = torch.zeros(nblk * stride, device=dev, dtype=torch.uint8)
    clen = torch.zeros(nblk, device=dev, dtype=torch.int32)
    B = L.batch
    N = nblk * bs
    t, med = timeit(lambda: B.compress_fast_batch_dev(src, soff, slen, comp, coff, ccap, clen, bs))
    C = int(clen.sum().item())
    if os.environ.get("COMPRESS_ONLY"):      # no room for a decompress buffer at the bench's 524 288 blocks: digest the streams
        h = torch.zeros(nblk, device=dev, dtype=torch.int64)
        B.xxh64_batch_dev(comp, coff, clen, h, 0)
        digest = int(h.sum().item()) & (2**64 - 1)
        print(f"compress: {N/t/2**30:.1f} GiB/s best ({N/med/2**30:.1f} med)  ratio {N/C:.3f}  streams {digest:016x}", flush=True)
        return
    out = torch.zeros(nblk * bs, device=dev, dtype=torch.uint8)
    res = torch.zeros(nblk, device=dev, dtype=torch.int32)
    out.zero_(); B.decompress_safe_batch_dev(comp, coff, clen, out, soff, slen, res)
    rt = bool((res == bs).all().item()) and bool(torch.equal(out, src))
    print(f"compress: {N/t/2**30:.1f} GiB/s best ({N/med/2**30:.1f} med)  ratio {N/C:.3f}  hbm {(N+C)/t/1e9:.0f} GB/s  roundtrip={rt}", flush=True)
    t, med = timeit(lambda: B.decompress_safe_batch_dev(comp, coff, clen, out, soff, slen, res))
    ok = bool((res == bs).all().item()) and bool(torch.equal(out, src))
    print(f"decompress_safe: {N/t/2**30:.1f} GiB/s best ({N/med/2**30:.1f} med) ok={ok}  hbm {(N+C)/t/1e9:.0f} GB/s", flush=True)
    out.zero_()
    t, med = timeit(lambda: B.decompress_fast_batch_dev(comp, coff, ccap, out, soff, slen, res))
    ok = bool((res == clen).all().item()) and bool(torch.equal(out, src))
    print(f"decompress_fast: {N/t/2**30:.1f} GiB/s best ({N/med/2**30:.1f} med) ok={ok}", flush=True)
    # xxh over 4 KiB buffers
    nb4 = N // 4096
    off4 = torch.arange(nb4, device=dev, dtype=torch.int64) * 4096
    len4 = torch.full((nb4,), 4096, device=dev, dtype=torch.int32)
    o64 = torch.zeros(nb4, device=dev, dtype=torch.int64); o32 = torch.zeros(nb4, device=dev, dtype=torch.int32)
    t, med = timeit(lambda: B.xxh64_batch_dev(src, off4, len4, o64, 0))
    print(f"xxh64 4KiB: {N/t/1e9:.0f} GB/s best ({N/med/1e9:.0f} med)", flush=True)
    t, med = timeit(lambda: B.xxh32_batch_dev(src, off4, len4, o32, 0))
    print(f"xxh32 4KiB: {N/t/1e9:.0f} GB/s best ({N/med/1e9:.0f} med)", flush=True)
    k = 12345 % nb4
    print("xxh64 check", int(o64[k].item()) & (2**64-1) == chk.xxh64(src[k*4096:(k+1)*4096].cpu().numpy(), 0))
    # xxh over 64 KiB blocks
    o64b = torch.zeros(nblk, device=dev, dtype=torch.int64)
    t, med = timeit(lambda: B.xxh64_batch_dev(src, soff, slen, o64b, 0))
    print(f"xxh64 64KiB: {N/t/1e9:.0f} GB/s best", flush=True)

if __name__ == "__main__" and not os.environ.get("HC"):
    main()


def hc_probe():
    """config 4 shape: 256 KiB blocks, HC level 9 — ratio vs the reference's LZ4_compress_HC(9) and GiB/s"""
    nblk = int(os.environ.get("HC_NBLK", 2048)); bs = 262144
    chk = O.best_available()
    base_n = min(nblk, 256)
    host = chk.datagen(base_n * bs, 0.5, 0.0, 4)
    dev = torch.device("cuda:0")
    src = torch.from_numpy(host).to(dev).repeat((nblk + base_n - 1) // base_n)[: nblk * bs].contiguous()
    bound = L.max_compressed_length(bs); stride = (bound + 15) // 16 * 16
    soff = torch.arange(nblk, device=dev, dtype=torch.int64) * bs
    slen = torch.full((nblk,), bs, device=dev, dtype=torch.int32)
    coff = torch.arange(nblk, device=dev, dtype=torch.int64) * stride
    ccap = torch.full((nblk,), bound, device=dev, dtype=torch.int32)
    comp = torch.zeros(nblk * stride, device=dev, dtype=torch.uint8)
    clen = torch.zeros(nblk, device=dev, dtype=torch.int32)
    t, med = timeit(lambda: L.batch.compress_hc_batch_dev(src, soff, slen, comp, coff, ccap, clen, 9), iters=2, warm=1)
    N = nblk * bs; C = int(clen.sum().item())
    ref_c = sum(len(chk.compress_hc(host[i * bs:(i + 1) * bs], 9)) for i in range(4)) if hasattr(chk, "compress_hc") else 0
    gpu_c4 = int(clen[:4].sum().item())
    print(f"HC-9 256KiB x{nblk}: {N/t/2**30:.2f} GiB/s  ratio {N/C:.3f}  (first 4 blocks: ours {4*bs/gpu_c4:.3f} vs reference HC-9 {4*bs/max(ref_c,1):.3f})", flush=True)
    out = torch.zeros(nblk * bs, device=dev, dtype=torch.uint8); res = torch.zeros(nblk, device=dev, dtype=torch.int32)
    L.batch.decompress_safe_batch_dev(comp, coff, clen, out, soff, slen, res)
    print("HC roundtrip ok:", bool((res == bs).all().item()) and bool(torch.equal(out, src)), flush=True)


if __name__ == "__main__" and os.environ.get("HC"):
    hc_probe()
