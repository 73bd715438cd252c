// common.cuh — warp-level helpers shared by the sm_90a kernels of libb200lz4.
//
// Everything here is byte/integer work: no tensor cores, no floating point.  A "block" in this
// library is an LZ4 block (an independent unit of 0..4 MiB), not a CUDA thread block; CUDA thread
// blocks are called CTAs.
#pragma once
#include <cstdint>
#ifdef B200_HOST_SIM            // tests/simt: the same kernel source run by a CPU SIMT emulator (test infrastructure only)
#include "simt.h"
#else
#include <cuda_runtime.h>
#endif

#define B200_FULL 0xFFFFFFFFu

// The few things that are PTX or CUDA-only syntax go through these, so that tests/simt can run the same source.
#ifdef B200_HOST_SIM
#define B200_DYN_SMEM(name, al) uint8_t* name = simt::dyn_smem()
#define B200_PREFETCH_L2(ptr) ((void)(ptr))
#define B200_PREFETCH_L1(ptr) ((void)(ptr))
#define B200_NANOSLEEP(ns) ((void)(ns))
#else
#define B200_DYN_SMEM(name, al) extern __shared__ __align__(al) uint8_t name[]
#define B200_PREFETCH_L2(ptr) asm volatile("prefetch.global.L2 [%0];" :: "l"(__cvta_generic_to_global(ptr)))
#define B200_PREFETCH_L1(ptr) asm volatile("prefetch.global.L1 [%0];" :: "l"(__cvta_generic_to_global(ptr)))
#define B200_NANOSLEEP(ns) __nanosleep(ns)
#endif

// A kernel launch that the emulator build runs as well: <<<grid, block, 0, st>>> on the GPU, one CTA after the other there.
#ifdef B200_HOST_SIM
#define B200_LAUNCH(kernel, grid, block, st, ...) simt::launch((unsigned)(grid), (block), [&] { kernel(__VA_ARGS__); })
#else
#define B200_LAUNCH(kernel, grid, block, st, ...) kernel<<<(grid), (block), 0, (st)>>>(__VA_ARGS__)
#endif

namespace b200 {

__device__ __forceinline__ int lane_id() { return threadIdx.x & 31; }

// Little-endian 32-bit load from an arbitrarily aligned address: two aligned word loads and a
// funnel shift.  Touches only aligned words that contain at least one requested byte, so it can
// never cross into an unmapped page beyond the caller's buffer.
__device__ __forceinline__ uint32_t load_u32_unaligned(const uint8_t* p)
{
    const uintptr_t a = reinterpret_cast<uintptr_t>(p);
    const uint32_t* w = reinterpret_cast<const uint32_t*>(a & ~uintptr_t(3));
    const uint32_t sh = (uint32_t(a) & 3u) * 8u;
    uint32_t lo = w[0];
    if (sh == 0) return lo;
    uint32_t hi = w[1];
    return __funnelshift_r(lo, hi, sh);
}

// Byte load that bypasses L1 (served by L2): used for LZ4 match sources, i.e. bytes this warp wrote
// moments ago.  Stores are write-through to L2, so L2 is where the data is; skipping L1 also keeps
// the scattered look-back lines from evicting the sequential input stream.
__device__ __forceinline__ uint8_t load_u8_l2(const uint8_t* p)
{
#ifdef B200_HOST_SIM
    return *p;
#else
    uint32_t v;
    asm volatile("ld.global.cg.u8 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return uint8_t(v);
#endif
}

// Cooperative copy of n bytes between NON-overlapping ranges (or ranges whose distance is at
// least the copy length).  32 lanes, 4 bytes per lane per iteration once dst is word-aligned.
// `sync_each_iter` inserts a warp barrier between iterations: required when dst-src < n but
// >= 128 (an LZ4 match whose period is at least one full iteration), so that iteration k reads
// what iteration k-1 wrote.
template <bool SYNC_EACH_ITER>
__device__ __forceinline__ void warp_copy_words(uint8_t* d, const uint8_t* s, int n, int lane)
{
    int head = int((0u - uint32_t(reinterpret_cast<uintptr_t>(d))) & 3u);
    if (head > n) head = n;
    if (lane < head) d[lane] = s[lane];
    d += head; s += head; n -= head;
    const int nw = n >> 2;
    const uintptr_t sa = reinterpret_cast<uintptr_t>(s);
    const uint32_t* sw = reinterpret_cast<const uint32_t*>(sa & ~uintptr_t(3));
    const uint32_t sh = (uint32_t(sa) & 3u) * 8u;
    uint32_t* dw = reinterpret_cast<uint32_t*>(d);
    if (SYNC_EACH_ITER) __syncwarp();
    for (int base = 0; base < nw; base += 32) {
        const int w = base + lane;
        if (w < nw) {
            uint32_t v = sw[w];
            if (sh) v = __funnelshift_r(v, sw[w + 1], sh);
            dw[w] = v;
        }
        if (SYNC_EACH_ITER) __syncwarp();
    }
    const int tail = n & 3;
    if (lane < tail) d[nw * 4 + lane] = s[nw * 4 + lane];
}

// Copy n bytes, any n: one predicated byte per lane when n <= 32, words otherwise.
__device__ __forceinline__ void warp_copy(uint8_t* d, const uint8_t* s, int n, int lane)
{
    if (n <= 32) { if (lane < n) d[lane] = s[lane]; }
    else warp_copy_words<false>(d, s, n, lane);
}

// LZ4 match copy: dst[op+i] = dst[op+i-off] for i in [0,ml), byte-serial semantics
// (lz4_Block_format.md "overlap"), executed by 32 lanes.  The caller has already issued a warp
// barrier after the last store into dst.  off >= 1.
__device__ __forceinline__ void warp_match_copy(uint8_t* dst_op, int off, int ml, int lane)
{
    const uint8_t* m = dst_op - off;
    if (off >= ml) {                       // disjoint: plain copy
        warp_copy(dst_op, m, ml, lane);
    } else if (off >= 128) {               // period >= one word-iteration: iterate with barriers
        warp_copy_words<true>(dst_op, m, ml, lane);
    } else if (off >= 32) {                // period >= one byte-iteration
        for (int base = 0; base < ml; base += 32) {
            const int i = base + lane;
            if (i < ml) dst_op[i] = m[i];
            __syncwarp();
        }
    } else {                               // short period: every byte comes from the first period,
        int r = lane % off;                // which already exists before op
        const int step = 32 % off;
        for (int base = 0; base < ml; base += 32) {
            const int i = base + lane;
            if (i < ml) dst_op[i] = m[r];
            r += step; if (r >= off) r -= off;
        }
    }
}

} // namespace b200
