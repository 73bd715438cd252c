// xxhash.cu — batch XXH32 / XXH64 (xxHash 0.6.5 semantics), one buffer per lane.
//
// Replaces the reference's XXH32 / XXH64 one-shots (xxhash.c:392-416 -> 351-389, 855-879 ->
// 810-852; JNI call sites src/jni/net_jpountz_xxhash_XXHashJNI.c:54,78,164,188) and the streaming
// state machine (xxhash.c:437-563, 898-1016; JNI :89-145, :199-255).  Bit-exact.
//
// The stripe loop of one buffer is a serial chain per accumulator (acc = rotl(acc + w*P2, r) * P1),
// so the parallelism is across buffers: every lane owns one buffer and keeps the four accumulators
// in registers (4-way ILP).  The loads are the problem: lane-per-buffer reads are strided by the
// buffer size, so instead each warp streams its 32 buffers through shared memory with TMA bulk
// copies (cp.async.bulk.shared.global, one per lane and chunk, completion on a per-warp mbarrier,
// two stages): HBM sees full-line sequential reads, lanes read their own slot with conflict-free
// 16-byte LDS (slot stride CHUNK+16).  Buffers that are not 16-byte aligned take a direct-load path.
//
// Algorithmic HBM bytes per buffer: len + 4 (XXH32) / len + 8 (XXH64).
#include "common.cuh"
#include "kernels.h"

namespace b200 {

static constexpr uint32_t P32_1 = 2654435761u, P32_2 = 2246822519u, P32_3 = 3266489917u,
                          P32_4 = 668265263u, P32_5 = 374761393u;
static constexpr uint64_t P64_1 = 11400714785074694791ull, P64_2 = 14029467366897019727ull,
                          P64_3 = 1609587929392839161ull, P64_4 = 9650029242287828579ull,
                          P64_5 = 2870177450012600261ull;

__device__ __forceinline__ uint32_t rotl32(uint32_t x, int r) { return __funnelshift_l(x, x, r); }
__device__ __forceinline__ uint64_t rotl64(uint64_t x, int r) { return (x << r) | (x >> (64 - r)); }
__device__ __forceinline__ uint32_t round32(uint32_t acc, uint32_t w) { return rotl32(acc + w * P32_2, 13) * P32_1; }  // xxhash.c:269-275
__device__ __forceinline__ uint64_t round64(uint64_t acc, uint64_t w) { return rotl64(acc + w * P64_2, 31) * P64_1; }  // xxhash.c:672-678
__device__ __forceinline__ uint64_t merge64(uint64_t h, uint64_t v) { return (h ^ round64(0, v)) * P64_1 + P64_4; }    // xxhash.c:680-686

__device__ __forceinline__ uint64_t load_u64_unaligned(const uint8_t* p)
{
    return uint64_t(load_u32_unaligned(p)) | (uint64_t(load_u32_unaligned(p + 4)) << 32);
}

// xxhash.c:290-348 (tail of < 16 bytes, then avalanche :278-286)
__device__ __forceinline__ uint32_t finish32(uint32_t h, const uint8_t* p, uint32_t rem)
{
    while (rem >= 4) { h = rotl32(h + load_u32_unaligned(p) * P32_3, 17) * P32_4; p += 4; rem -= 4; }
    while (rem)      { h = rotl32(h + uint32_t(*p++) * P32_5, 11) * P32_1; rem--; }
    h ^= h >> 15; h *= P32_2; h ^= h >> 13; h *= P32_3; h ^= h >> 16;
    return h;
}
// xxhash.c:701-808 (tail of < 32 bytes, then avalanche :688-696)
__device__ __forceinline__ uint64_t finish64(uint64_t h, const uint8_t* p, uint32_t rem)
{
    while (rem >= 8) { h = rotl64(h ^ round64(0, load_u64_unaligned(p)), 27) * P64_1 + P64_4; p += 8; rem -= 8; }
    if (rem >= 4)    { h = rotl64(h ^ (uint64_t(load_u32_unaligned(p)) * P64_1), 23) * P64_2 + P64_3; p += 4; rem -= 4; }
    while (rem)      { h = rotl64(h ^ (uint64_t(*p++) * P64_5), 11) * P64_1; rem--; }
    h ^= h >> 33; h *= P64_2; h ^= h >> 29; h *= P64_3; h ^= h >> 32;
    return h;
}

#ifndef B200_HOST_SIM          // PTX: not part of the emulated build (tests/simt)
// ---- mbarrier / TMA bulk-copy primitives (PTX; SASS: SYNCS.*, UBLKCP)
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count)
{ asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(bar), "r"(count) : "memory"); }
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes)
{ asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(bar), "r"(bytes) : "memory"); }
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity)
{
    uint32_t ok;
    do {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
    } while (!ok);
}
__device__ __forceinline__ void tma_bulk_g2s(uint32_t dst_smem, const void* src_gmem, uint32_t bytes, uint32_t bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 :: "r"(dst_smem), "l"(src_gmem), "r"(bytes), "r"(bar) : "memory");
}

#endif

template <int BITS> struct XxhTraits;
template <> struct XxhTraits<32> { using word = uint32_t; static constexpr int STRIPE = 16; };
template <> struct XxhTraits<64> { using word = uint64_t; static constexpr int STRIPE = 32; };

template <int BITS> struct Acc;
template <> struct Acc<32> {
    uint32_t v1, v2, v3, v4;
    __device__ __forceinline__ void init(uint32_t seed) { v1 = seed + P32_1 + P32_2; v2 = seed + P32_2; v3 = seed; v4 = seed - P32_1; }
    __device__ __forceinline__ void stripe(uint4 q) { v1 = round32(v1, q.x); v2 = round32(v2, q.y); v3 = round32(v3, q.z); v4 = round32(v4, q.w); }
    __device__ __forceinline__ void stripe_g(const uint8_t* p) {
        stripe(make_uint4(load_u32_unaligned(p), load_u32_unaligned(p + 4), load_u32_unaligned(p + 8), load_u32_unaligned(p + 12)));
    }
    __device__ __forceinline__ uint32_t merge() const { return rotl32(v1, 1) + rotl32(v2, 7) + rotl32(v3, 12) + rotl32(v4, 18); }
};
template <> struct Acc<64> {
    uint64_t v1, v2, v3, v4;
    __device__ __forceinline__ void init(uint64_t seed) { v1 = seed + P64_1 + P64_2; v2 = seed + P64_2; v3 = seed; v4 = seed - P64_1; }
    __device__ __forceinline__ void stripe(uint4 a, uint4 b) {
        v1 = round64(v1, uint64_t(a.x) | (uint64_t(a.y) << 32)); v2 = round64(v2, uint64_t(a.z) | (uint64_t(a.w) << 32));
        v3 = round64(v3, uint64_t(b.x) | (uint64_t(b.y) << 32)); v4 = round64(v4, uint64_t(b.z) | (uint64_t(b.w) << 32));
    }
    __device__ __forceinline__ void stripe_g(const uint8_t* p) {
        v1 = round64(v1, load_u64_unaligned(p)); v2 = round64(v2, load_u64_unaligned(p + 8));
        v3 = round64(v3, load_u64_unaligned(p + 16)); v4 = round64(v4, load_u64_unaligned(p + 24));
    }
    __device__ __forceinline__ uint64_t merge() const {
        uint64_t h = rotl64(v1, 1) + rotl64(v2, 7) + rotl64(v3, 12) + rotl64(v4, 18);
        h = merge64(h, v1); h = merge64(h, v2); h = merge64(h, v3); h = merge64(h, v4);
        return h;
    }
};

#ifndef B200_HOST_SIM          // TMA-staged batch kernel and its launchers: CUDA only
static constexpr int XXH_WARPS = 4;
static constexpr int XXH_CHUNK = 256;                    // bytes per lane per stage
static constexpr int XXH_SLOT  = XXH_CHUNK + 16;         // slot stride: 16-byte LDS conflict-free
static constexpr int XXH_STAGES = 2;
static constexpr size_t XXH_SMEM = size_t(XXH_WARPS) * XXH_STAGES * 32 * XXH_SLOT + 64;

template <int BITS>
__global__ void __launch_bounds__(XXH_WARPS * 32)
xxh_batch_kernel(const uint8_t* __restrict__ base, const uint64_t* __restrict__ off, const int32_t* __restrict__ len,
                 typename XxhTraits<BITS>::word seed, typename XxhTraits<BITS>::word* __restrict__ out, uint32_t n)
{
    using word = typename XxhTraits<BITS>::word;
    constexpr int STRIPE = XxhTraits<BITS>::STRIPE;
    extern __shared__ __align__(128) uint8_t smem[];
    const int warp = threadIdx.x >> 5, lane = lane_id();
    const uint32_t first = (blockIdx.x * XXH_WARPS + warp) * 32;
    if (first >= n) return;
    const uint32_t i = first + lane;
    const bool live = i < n;

    const uint8_t* p = live ? base + off[i] : base;
    const uint32_t L = live ? (uint32_t)max(len[i], 0) : 0u;
    const uint32_t bulk = L & ~uint32_t(STRIPE - 1);                // whole stripes
    Acc<BITS> acc; acc.init(seed);

    uint64_t* bars = reinterpret_cast<uint64_t*>(smem);             // XXH_WARPS * XXH_STAGES mbarriers
    uint8_t* slots = smem + 64 + size_t(warp) * XXH_STAGES * 32 * XXH_SLOT;
    const bool aligned = (reinterpret_cast<uintptr_t>(p) & 15) == 0 || bulk == 0;

    if (__all_sync(B200_FULL, aligned)) {
        const uint32_t bar0 = smem_u32(&bars[warp * XXH_STAGES]);
        if (lane == 0) {
            for (int s = 0; s < XXH_STAGES; s++) mbar_init(bar0 + 8 * s, 1);
            asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        }
        __syncwarp();
        const uint32_t nchunks = (bulk + XXH_CHUNK - 1) / XXH_CHUNK;
        const uint32_t maxchunks = __reduce_max_sync(B200_FULL, nchunks);

        auto issue = [&](uint32_t k) {                              // chunk k -> stage k % STAGES
            const uint32_t s = k % XXH_STAGES;
            const uint32_t bytes = k < nchunks ? min(uint32_t(XXH_CHUNK), bulk - k * XXH_CHUNK) : 0u;
            const uint32_t total = __reduce_add_sync(B200_FULL, bytes);
            if (lane == 0) mbar_arrive_expect_tx(bar0 + 8 * s, total);
            if (bytes) tma_bulk_g2s(smem_u32(slots + (size_t(s) * 32 + lane) * XXH_SLOT), p + size_t(k) * XXH_CHUNK, bytes, bar0 + 8 * s);
        };
        for (uint32_t k = 0; k < XXH_STAGES && k < maxchunks; k++) issue(k);
        for (uint32_t k = 0; k < maxchunks; k++) {
            const uint32_t s = k % XXH_STAGES;
            mbar_wait(bar0 + 8 * s, (k / XXH_STAGES) & 1);
            if (k < nchunks) {
                const uint32_t bytes = min(uint32_t(XXH_CHUNK), bulk - k * XXH_CHUNK);
                const uint4* q = reinterpret_cast<const uint4*>(slots + (size_t(s) * 32 + lane) * XXH_SLOT);
                if constexpr (BITS == 32) {
                    #pragma unroll 4
                    for (uint32_t j = 0; j < bytes / 16; j++) acc.stripe(q[j]);
                } else {
                    #pragma unroll 4
                    for (uint32_t j = 0; j < bytes / 32; j++) acc.stripe(q[2 * j], q[2 * j + 1]);
                }
            }
            __syncwarp();                                           // every lane is done with stage s
            if (k + XXH_STAGES < maxchunks) issue(k + XXH_STAGES);
        }
    } else {
        for (uint32_t o = 0; o < bulk; o += STRIPE) acc.stripe_g(p + o);
    }

    if (live) {
        if constexpr (BITS == 32) {
            uint32_t h = (L >= 16u) ? acc.merge() : seed + P32_5;
            out[i] = finish32(h + L, p + bulk, L - bulk);
        } else {
            uint64_t h = (L >= 32u) ? acc.merge() : seed + P64_5;
            out[i] = finish64(h + uint64_t(L), p + bulk, L - bulk);
        }
    }
}

cudaError_t launch_xxh32(const uint8_t* base, const uint64_t* off, const int32_t* len, uint32_t seed,
                         uint32_t* out, size_t n, cudaStream_t st)
{
    if (n == 0) return cudaSuccess;
    auto k = xxh_batch_kernel<32>;
    cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)XXH_SMEM);
    if (e != cudaSuccess) return e;
    const unsigned grid = (unsigned)((n + XXH_WARPS * 32 - 1) / (XXH_WARPS * 32));
    k<<<grid, XXH_WARPS * 32, XXH_SMEM, st>>>(base, off, len, seed, out, (uint32_t)n);
    return cudaGetLastError();
}

cudaError_t launch_xxh64(const uint8_t* base, const uint64_t* off, const int32_t* len, uint64_t seed,
                         uint64_t* out, size_t n, cudaStream_t st)
{
    if (n == 0) return cudaSuccess;
    auto k = xxh_batch_kernel<64>;
    cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)XXH_SMEM);
    if (e != cudaSuccess) return e;
    const unsigned grid = (unsigned)((n + XXH_WARPS * 32 - 1) / (XXH_WARPS * 32));
    k<<<grid, XXH_WARPS * 32, XXH_SMEM, st>>>(base, off, len, seed, out, (uint32_t)n);
    return cudaGetLastError();
}

#endif

// ------------------------------------------------------------------ one long XXH32 stream per warp
// A single XXH32 stream is four serial accumulator chains (xxhash.c:269-275: acc = rotl(acc + w*P2, 13) * P1,
// ~10 cycles per 16-byte stripe), so one stream cannot go faster than ~3 GB/s on this clock whatever feeds it.
// The batch kernel above gives every lane its own buffer — right for millions of small buffers, wrong for a
// handful of large ones (32 frames of 64 MiB would sit in ONE warp).  Here a whole warp feeds one stream:
// rows of 128 bytes are loaded coalesced (one word per lane), two groups of 8 rows in flight, and every lane
// runs chain (lane & 3) on words pulled out of the row registers by shuffle (word j of stripe s sits in lane
// 4*s + j).  All eight lane quads compute the same four chains, so the result is valid on every lane.
// Long streams then scale with the number of streams: one warp (one SM) each.
__device__ __forceinline__ uint32_t xxh32_chain_init(uint32_t seed, int lane)
{
    const int c = lane & 3;
    return c == 0 ? seed + P32_1 + P32_2 : c == 1 ? seed + P32_2 : c == 2 ? seed : seed - P32_1;
}

// Consume `rows` rows of 128 bytes starting at p (any alignment) into this lane's chain.  CG: the bytes are being produced by
// ANOTHER kernel while this one runs (the frame variant below) -- every load then goes to L2 (ld.global.cg); a line this SM's
// L1 took earlier may predate a neighbouring block's bytes.
template <bool CG>
__device__ __forceinline__ uint32_t xxh_ldw(const uint32_t* p)
{
#ifndef B200_HOST_SIM
    if constexpr (CG) return __ldcg(p);
#endif
    return *p;
}

template <bool CG = false>
__device__ __forceinline__ uint32_t xxh32_warp_rows(uint32_t v, const uint8_t* __restrict__ p, size_t rows, int lane)
{
    constexpr int R = 8;
    const uintptr_t sa = reinterpret_cast<uintptr_t>(p);
    const uint32_t* __restrict__ W = reinterpret_cast<const uint32_t*>(sa & ~uintptr_t(3));
    const uint32_t sh = (uint32_t(sa) & 3u) * 8u;
    const int c = lane & 3;
    auto ldrow = [&](size_t r) -> uint32_t {
        const size_t i = r * 32 + lane;
        const uint32_t a = xxh_ldw<CG>(W + i);
        return sh ? __funnelshift_r(a, xxh_ldw<CG>(W + i + 1), sh) : a;
    };
    uint32_t cur[R], nxt[R];
    const size_t groups = rows / R;
    if (groups) {
        #pragma unroll
        for (int r = 0; r < R; r++) cur[r] = ldrow(r);
    }
    for (size_t g = 0; g < groups; g++) {
        if (g + 1 < groups) {
            #pragma unroll
            for (int r = 0; r < R; r++) nxt[r] = ldrow((g + 1) * R + r);
        }
        #pragma unroll
        for (int r = 0; r < R; r++) {
            #pragma unroll
            for (int st = 0; st < 8; st++) v = round32(v, __shfl_sync(B200_FULL, cur[r], 4 * st + c));
        }
        #pragma unroll
        for (int r = 0; r < R; r++) cur[r] = nxt[r];
    }
    for (size_t r = groups * R; r < rows; r++) {
        const uint32_t x = ldrow(r);
        #pragma unroll
        for (int st = 0; st < 8; st++) v = round32(v, __shfl_sync(B200_FULL, x, 4 * st + c));
    }
    return v;
}

// All stripes of [p, p + 16*stripes): rows by the warp, the last < 8 stripes by direct loads.
template <bool CG = false>
__device__ __forceinline__ uint32_t xxh32_warp_stripes(uint32_t v, const uint8_t* __restrict__ p, size_t stripes, int lane)
{
    const size_t rows = stripes >> 3;
    v = xxh32_warp_rows<CG>(v, p, rows, lane);
    for (size_t t = rows << 3; t < stripes; t++) {
        const uint8_t* q = p + 16 * t + 4 * (lane & 3);
        if constexpr (CG) {
            const uintptr_t a = reinterpret_cast<uintptr_t>(q);
            const uint32_t* w = reinterpret_cast<const uint32_t*>(a & ~uintptr_t(3));
            const uint32_t sh = (uint32_t(a) & 3u) * 8u;
            const uint32_t lo = xxh_ldw<true>(w);
            v = round32(v, sh ? __funnelshift_r(lo, xxh_ldw<true>(w + 1), sh) : lo);
        } else {
            v = round32(v, load_u32_unaligned(q));
        }
    }
    return v;
}

__device__ __forceinline__ uint32_t xxh32_chain_merge(uint32_t v)
{
    return rotl32(__shfl_sync(B200_FULL, v, 0), 1) + rotl32(__shfl_sync(B200_FULL, v, 1), 7) +
           rotl32(__shfl_sync(B200_FULL, v, 2), 12) + rotl32(__shfl_sync(B200_FULL, v, 3), 18);
}

__global__ void __launch_bounds__(32)
xxh32_long_kernel(const uint8_t* __restrict__ base, const uint64_t* __restrict__ off, const int32_t* __restrict__ len,
                  uint32_t seed, uint32_t* __restrict__ out, uint32_t n)
{
    const uint32_t i = blockIdx.x;
    if (i >= n) return;
    const int lane = lane_id();
    const uint8_t* __restrict__ p = base + off[i];
    const uint32_t L = (uint32_t)max(len[i], 0);
    const size_t stripes = L >> 4;
    uint32_t h;
    if (L >= 16u) h = xxh32_chain_merge(xxh32_warp_stripes(xxh32_chain_init(seed, lane), p, stripes, lane));
    else h = seed + P32_5;
    if (lane == 0) out[i] = finish32(h + L, p + 16 * stripes, L & 15u);
}

#ifndef B200_HOST_SIM
cudaError_t launch_xxh32_long(const uint8_t* base, const uint64_t* off, const int32_t* len, uint32_t seed,
                              uint32_t* out, size_t n, cudaStream_t st)
{
    if (n == 0) return cudaSuccess;
    xxh32_long_kernel<<<(unsigned)n, 32, 0, st>>>(base, off, len, seed, out, (uint32_t)n);
    return cudaGetLastError();
}
#endif

// xxh32_long_kernel (seed 0) for one run of a stream that goes on from call to call (the incremental frame writer): 64-bit
// lengths, and the state carried in and out (XXH_CARRY_*).  The bytes of an unfinished stripe (a run that ends inside one,
// after a flushed short block or a WRITE that stopped mid-stripe) wait in the state for the next run; a run that does not
// complete the stripe only adds to them.
__global__ void __launch_bounds__(32)
xxh32_long_carry_kernel(const uint8_t* __restrict__ base, const uint64_t* __restrict__ off, const uint64_t* __restrict__ len,
                        uint32_t* __restrict__ out, Xxh32Carry* __restrict__ c_state, const uint8_t* __restrict__ c_mode, uint32_t n)
{
    __shared__ __align__(16) uint8_t s_mem[16];
    const uint32_t r = blockIdx.x;
    if (r >= n) return;
    const int lane = lane_id();
    const uint32_t mode = c_mode[r];
    const uint8_t* __restrict__ p = base + off[r];
    uint64_t L = len[r];
    uint32_t v = xxh32_chain_init(0u, lane), mem = 0;
    uint64_t total = 0;
    if (mode & XXH_CARRY_IN) {
        const Xxh32Carry& c = c_state[r];
        v = c.v[lane & 3]; total = c.total; mem = c.memsize;
        if (uint32_t(lane) < mem) s_mem[lane] = c.mem[lane];
    }
    __syncwarp();
    total += L;
    if (mem + L < 16u) {                                    // the stripe stays open
        if (uint32_t(lane) < L) s_mem[mem + lane] = p[lane];
        mem += (uint32_t)L; L = 0;
    } else {
        if (mem) {                                          // finish the stripe the previous run left open
            const uint32_t t = 16u - mem;
            if (uint32_t(lane) < t) s_mem[mem + lane] = p[lane];
            __syncwarp();
            v = round32(v, reinterpret_cast<const uint32_t*>(s_mem)[lane & 3]);
            p += t; L -= t; mem = 0;
            __syncwarp();
        }
        const size_t stripes = size_t(L >> 4);
        v = xxh32_warp_stripes(v, p, stripes, lane);
        mem = uint32_t(L & 15u);
        if (uint32_t(lane) < mem) s_mem[lane] = p[16 * stripes + lane];
    }
    __syncwarp();
    if (mode & XXH_CARRY_OUT) {
        Xxh32Carry& c = c_state[r];
        if (lane < 4) c.v[lane] = v;
        if (uint32_t(lane) < mem) c.mem[lane] = s_mem[lane];
        if (lane == 0) { c.total = total; c.memsize = mem; }
        return;
    }
    const uint32_t h = total >= 16 ? xxh32_chain_merge(v) : 0u + P32_5;
    if (lane == 0) out[r] = finish32(h + uint32_t(total), s_mem, mem);
}

cudaError_t launch_xxh32_long_carry(const uint8_t* base, const uint64_t* off, const uint64_t* len, uint32_t* out, Xxh32Carry* carry,
                                    const uint8_t* mode, size_t n, cudaStream_t st)
{
    if (n == 0) return cudaSuccess;
    B200_LAUNCH(xxh32_long_carry_kernel, (unsigned)n, 32, st, base, off, len, out, carry, mode, (uint32_t)n);
    return cudaGetLastError();
}

// ------------------------------------------------------------------ frame content checksums, chained to the block decoder
// LZ4FrameInputStream verifies a frame's content XXH32 after its last block (LZ4FrameInputStream.java:264-273).  As a
// second pass over 32 frames of 64 MiB it costs as much as decoding them (a stream is four serial chains, ~3 GB/s, however
// many SMs idle).  Here one warp per frame runs WHILE the blocks are decoded (another stream, same device): it takes the
// frame's blocks in order, spins on the decoder's per-block result word until that block is there (the decoder publishes it
// behind a __threadfence), and folds the block in.  The decode kernel is launched first and never waits for this one.
//   blk_off[b]: where block b lies in the slot layout;  blk_comp[b] >= 0: its index in the decoder's result array;  < 0: a
//   stored block of blk_rawlen[b] bytes, already in place.  c_res[k] == FRAME_RES_PENDING until block k is decoded; a negative
//   result ends the frame's hash (the host reports -6).  Blocks need not be full: the bytes of an unfinished 16-byte stripe
//   wait in shared memory for the next block (a frame written with flush() calls has short blocks anywhere).  Short blocks
//   share 32-byte sectors with their neighbours, which may be written after this warp looked at the sector: block bytes are
//   read with ld.global.cg (L2), never through this SM's L1.
__device__ __forceinline__ uint8_t ld_byte_l2(const uint8_t* p)
{
#ifndef B200_HOST_SIM
    return __ldcg(p);
#else
    return *p;
#endif
}

__global__ void __launch_bounds__(32)
xxh32_frames_chained_kernel(const uint8_t* __restrict__ slots, const uint64_t* __restrict__ blk_off, const uint32_t* __restrict__ f_first,
                            const uint32_t* __restrict__ f_nblk, const int32_t* __restrict__ blk_comp, const int32_t* __restrict__ blk_rawlen,
                            const int32_t* c_res, uint32_t* __restrict__ out, uint32_t n, Xxh32Carry* c_state = nullptr,
                            const uint8_t* c_mode = nullptr)
{
    __shared__ __align__(16) uint8_t s_carry[16];
    const uint32_t f = blockIdx.x;
    if (f >= n) return;
    const int lane = lane_id();
    const uint32_t first = f_first[f], nblk = f_nblk[f];
    const uint32_t mode = c_mode ? c_mode[f] : 0u;          // XXH_CARRY_*: a frame that began or goes on in another call
    uint32_t v = xxh32_chain_init(0u, lane);
    uint64_t total = 0; uint32_t carry = 0;                 // bytes of the content seen so far; bytes waiting in s_carry
    bool big = false;                                       // at least one full stripe went through the chains
    if (mode & XXH_CARRY_IN) {
        const Xxh32Carry& c = c_state[f];
        v = c.v[lane & 3]; total = c.total; carry = c.memsize; big = total >= 16;
        if (uint32_t(lane) < carry) s_carry[lane] = c.mem[lane];
        __syncwarp();
    }
    for (uint32_t k = 0; k < nblk; k++) {
        const int32_t ci = blk_comp[first + k];
        int32_t r;
        if (ci < 0) r = blk_rawlen[first + k];
        else {
            const volatile int32_t* w = c_res + ci;
            r = 0;
            if (lane == 0) { while ((r = *w) == FRAME_RES_PENDING) { B200_NANOSLEEP(256); } }
            r = __shfl_sync(B200_FULL, r, 0);
            __threadfence();                                // the block's bytes were written before its result word
            if (r < 0) break;
        }
        const uint8_t* p = slots + blk_off[first + k];
        uint32_t len = uint32_t(r);
        total += len;
        if (carry) {                                        // finish the stripe the previous block left open
            const uint32_t t = min(16u - carry, len);
            if (uint32_t(lane) < t) s_carry[carry + lane] = ld_byte_l2(p + lane);
            __syncwarp();
            carry += t; p += t; len -= t;
            if (carry < 16u) continue;
            v = round32(v, reinterpret_cast<const uint32_t*>(s_carry)[lane & 3]); big = true; carry = 0;
            __syncwarp();
        }
        const size_t stripes = size_t(len) >> 4;
        if (stripes) { v = xxh32_warp_stripes<true>(v, p, stripes, lane); big = true; }
        carry = len & 15u;
        if (uint32_t(lane) < carry) s_carry[lane] = ld_byte_l2(p + 16 * stripes + lane);
        __syncwarp();
    }
    if (mode & XXH_CARRY_OUT) {                             // the frame goes on in a later call: its state, not its digest
        Xxh32Carry& c = c_state[f];
        if (lane < 4) c.v[lane] = v;
        if (uint32_t(lane) < carry) c.mem[lane] = s_carry[lane];
        if (lane == 0) { c.total = total; c.memsize = carry; }
        return;
    }
    const uint32_t h = big ? xxh32_chain_merge(v) : 0u + P32_5;
    if (lane == 0) out[f] = finish32(h + uint32_t(total), s_carry, carry);
}

#ifndef B200_HOST_SIM
cudaError_t launch_xxh32_frames_chained(const uint8_t* slots, const uint64_t* blk_off, const uint32_t* f_first, const uint32_t* f_nblk,
                                        const int32_t* blk_comp, const int32_t* blk_rawlen, const int32_t* c_res,
                                        uint32_t* out, size_t n, cudaStream_t st)
{
    if (n == 0) return cudaSuccess;
    xxh32_frames_chained_kernel<<<(unsigned)n, 32, 0, st>>>(slots, blk_off, f_first, f_nblk, blk_comp, blk_rawlen, c_res, out, (uint32_t)n);
    return cudaGetLastError();
}
#endif
// the incremental reader's launch (frame_reader.cu): the same code in the emulator build (B200_LAUNCH), where the decoder has
// finished before this runs and nothing spins
cudaError_t launch_xxh32_frames_chained_carry(const uint8_t* slots, const uint64_t* blk_off, const uint32_t* f_first,
                                              const uint32_t* f_nblk, const int32_t* blk_comp, const int32_t* blk_rawlen,
                                              const int32_t* c_res, uint32_t* out, size_t n, Xxh32Carry* carry,
                                              const uint8_t* mode, cudaStream_t st)
{
    if (n == 0) return cudaSuccess;
    B200_LAUNCH(xxh32_frames_chained_kernel, (unsigned)n, 32, st, slots, blk_off, f_first, f_nblk, blk_comp, blk_rawlen, c_res, out,
                (uint32_t)n, carry, mode);
    return cudaGetLastError();
}

// ---- the same for XXH64: stripes of 32 bytes, rows of 256 bytes (one 64-bit word per lane), chain = lane & 3.
__device__ __forceinline__ uint64_t xxh64_chain_init(uint64_t seed, int lane)
{
    const int c = lane & 3;
    return c == 0 ? seed + P64_1 + P64_2 : c == 1 ? seed + P64_2 : c == 2 ? seed : seed - P64_1;
}

__device__ __forceinline__ uint64_t xxh64_warp_rows(uint64_t v, const uint8_t* __restrict__ p, size_t rows, int lane)
{
    constexpr int R = 4;
    const uintptr_t sa = reinterpret_cast<uintptr_t>(p);
    const uint32_t* __restrict__ W = reinterpret_cast<const uint32_t*>(sa & ~uintptr_t(3));
    const uint32_t sh = (uint32_t(sa) & 3u) * 8u;
    const int c = lane & 3;
    auto ldrow = [&](size_t r) -> uint2 {
        const size_t i = (r * 32 + lane) * 2;
        const uint32_t a = W[i], b = W[i + 1];
        if (!sh) return make_uint2(a, b);
        return make_uint2(__funnelshift_r(a, b, sh), __funnelshift_r(b, W[i + 2], sh));
    };
    auto feed = [&](uint2 x) {
        #pragma unroll
        for (int st = 0; st < 8; st++) {
            const uint32_t lo = __shfl_sync(B200_FULL, x.x, 4 * st + c), hi = __shfl_sync(B200_FULL, x.y, 4 * st + c);
            v = round64(v, uint64_t(lo) | (uint64_t(hi) << 32));
        }
    };
    uint2 cur[R], nxt[R];
    const size_t groups = rows / R;
    if (groups) {
        #pragma unroll
        for (int r = 0; r < R; r++) cur[r] = ldrow(r);
    }
    for (size_t g = 0; g < groups; g++) {
        if (g + 1 < groups) {
            #pragma unroll
            for (int r = 0; r < R; r++) nxt[r] = ldrow((g + 1) * R + r);
        }
        #pragma unroll
        for (int r = 0; r < R; r++) feed(cur[r]);
        #pragma unroll
        for (int r = 0; r < R; r++) cur[r] = nxt[r];
    }
    for (size_t r = groups * R; r < rows; r++) feed(ldrow(r));
    return v;
}

__device__ __forceinline__ uint64_t xxh64_warp_stripes(uint64_t v, const uint8_t* __restrict__ p, size_t stripes, int lane)
{
    const size_t rows = stripes >> 3;
    v = xxh64_warp_rows(v, p, rows, lane);
    for (size_t t = rows << 3; t < stripes; t++) v = round64(v, load_u64_unaligned(p + 32 * t + 8 * (lane & 3)));
    return v;
}

__device__ __forceinline__ uint64_t shfl_u64(uint64_t x, int src)
{
    return uint64_t(__shfl_sync(B200_FULL, uint32_t(x), src)) | (uint64_t(__shfl_sync(B200_FULL, uint32_t(x >> 32), src)) << 32);
}

__device__ __forceinline__ uint64_t xxh64_chain_merge(uint64_t v)      // xxhash.c:792-802
{
    const uint64_t v1 = shfl_u64(v, 0), v2 = shfl_u64(v, 1), v3 = shfl_u64(v, 2), v4 = shfl_u64(v, 3);
    uint64_t h = rotl64(v1, 1) + rotl64(v2, 7) + rotl64(v3, 12) + rotl64(v4, 18);
    h = merge64(h, v1); h = merge64(h, v2); h = merge64(h, v3); h = merge64(h, v4);
    return h;
}

__global__ void __launch_bounds__(32)
xxh64_long_kernel(const uint8_t* __restrict__ base, const uint64_t* __restrict__ off, const int32_t* __restrict__ len,
                  uint64_t seed, uint64_t* __restrict__ out, uint32_t n)
{
    const uint32_t i = blockIdx.x;
    if (i >= n) return;
    const int lane = lane_id();
    const uint8_t* __restrict__ p = base + off[i];
    const uint32_t L = (uint32_t)max(len[i], 0);
    const size_t stripes = L >> 5;
    uint64_t h;
    if (L >= 32u) h = xxh64_chain_merge(xxh64_warp_stripes(xxh64_chain_init(seed, lane), p, stripes, lane));
    else h = seed + P64_5;
    if (lane == 0) out[i] = finish64(h + uint64_t(L), p + 32 * stripes, L & 31u);
}

#ifndef B200_HOST_SIM
cudaError_t launch_xxh64_long(const uint8_t* base, const uint64_t* off, const int32_t* len, uint64_t seed,
                              uint64_t* out, size_t n, cudaStream_t st)
{
    if (n == 0) return cudaSuccess;
    xxh64_long_kernel<<<(unsigned)n, 32, 0, st>>>(base, off, len, seed, out, (uint32_t)n);
    return cudaGetLastError();
}
#endif

// ------------------------------------------------------------------ streaming state (device-resident)
// One lane walks the XXH32_update / XXH64_update state machine (xxhash.c:515-546, 971-1002); the
// serial dependency makes more lanes pointless.  reset / digest are the same kernel with op codes.
__global__ void xxh32_stream_kernel(Xxh32State* s, int op, uint32_t seed, const uint8_t* __restrict__ p, size_t len)
{
    const int lane = lane_id();
    if (op == XXH_OP_RESET) {
        if (lane) return;
        s->total = 0; s->memsize = 0; s->seed = seed;
        s->v[0] = seed + P32_1 + P32_2; s->v[1] = seed + P32_2; s->v[2] = seed; s->v[3] = seed - P32_1;
        return;
    }
    if (op == XXH_OP_UPDATE) {
        // XXH32_update (xxhash.c:515-546) with the stripe loop spread over the warp (xxh32_warp_stripes); the state is
        // read by every lane (uniform control flow) and written back by lanes 0-3 / lane 0.
        const uint32_t memsize = s->memsize;
        const uint64_t total = s->total;
        uint32_t v = s->v[lane & 3];
        __syncwarp();
        if (memsize + len < 16) {
            if (lane == 0) { for (size_t i = 0; i < len; i++) s->mem[memsize + i] = p[i]; s->memsize = memsize + (uint32_t)len; s->total = total + len; }
            return;
        }
        if (memsize) {
            const uint32_t fill = 16 - memsize;
            if (lane == 0) for (uint32_t i = 0; i < fill; i++) s->mem[memsize + i] = p[i];
            __syncwarp();
            v = round32(v, load_u32_unaligned(s->mem + 4 * (lane & 3)));
            p += fill; len -= fill;
            __syncwarp();
        }
        const size_t stripes = len >> 4;
        v = xxh32_warp_stripes(v, p, stripes, lane);
        if (lane < 4) s->v[lane] = v;
        if (lane == 0) {
            const uint32_t r = (uint32_t)(len & 15);
            for (uint32_t i = 0; i < r; i++) s->mem[i] = p[16 * stripes + i];
            s->memsize = r; s->total = total + (memsize ? 16 - memsize : 0) + len;
        }
        return;
    }
    if (lane) return;
    {   // digest (xxhash.c:548-563): non-destructive
        uint32_t h;
        if (s->total >= 16) h = rotl32(s->v[0], 1) + rotl32(s->v[1], 7) + rotl32(s->v[2], 12) + rotl32(s->v[3], 18);
        else h = s->seed + P32_5;
        h += (uint32_t)s->total;
        s->digest = finish32(h, s->mem, s->memsize);
    }
}

__global__ void xxh64_stream_kernel(Xxh64State* s, int op, uint64_t seed, const uint8_t* __restrict__ p, size_t len)
{
    const int lane = lane_id();
    if (op == XXH_OP_RESET) {
        if (lane) return;
        s->total = 0; s->memsize = 0; s->seed = seed;
        s->v[0] = seed + P64_1 + P64_2; s->v[1] = seed + P64_2; s->v[2] = seed; s->v[3] = seed - P64_1;
        return;
    }
    if (op == XXH_OP_UPDATE) {                               // XXH64_update (xxhash.c:971-1002), stripe loop by the warp
        const uint32_t memsize = s->memsize;
        const uint64_t total = s->total;
        uint64_t v = s->v[lane & 3];
        __syncwarp();
        if (memsize + len < 32) {
            if (lane == 0) { for (size_t i = 0; i < len; i++) s->mem[memsize + i] = p[i]; s->memsize = memsize + (uint32_t)len; s->total = total + len; }
            return;
        }
        if (memsize) {
            const uint32_t fill = 32 - memsize;
            if (lane == 0) for (uint32_t i = 0; i < fill; i++) s->mem[memsize + i] = p[i];
            __syncwarp();
            v = round64(v, load_u64_unaligned(s->mem + 8 * (lane & 3)));
            p += fill; len -= fill;
            __syncwarp();
        }
        const size_t stripes = len >> 5;
        v = xxh64_warp_stripes(v, p, stripes, lane);
        if (lane < 4) s->v[lane] = v;
        if (lane == 0) {
            const uint32_t r = (uint32_t)(len & 31);
            for (uint32_t i = 0; i < r; i++) s->mem[i] = p[32 * stripes + i];
            s->memsize = r; s->total = total + (memsize ? 32 - memsize : 0) + len;
        }
        return;
    }
    if (lane) return;
    {
        uint64_t h;
        if (s->total >= 32) {
            h = rotl64(s->v[0], 1) + rotl64(s->v[1], 7) + rotl64(s->v[2], 12) + rotl64(s->v[3], 18);
            for (int k = 0; k < 4; k++) h = merge64(h, s->v[k]);
        } else h = s->seed + P64_5;
        h += s->total;
        s->digest = finish64(h, s->mem, s->memsize);
    }
}

#ifndef B200_HOST_SIM
cudaError_t launch_xxh32_stream(Xxh32State* st, int op, uint32_t seed, const uint8_t* data, size_t len, cudaStream_t s)
{
    xxh32_stream_kernel<<<1, 32, 0, s>>>(st, op, seed, data, len);
    return cudaGetLastError();
}
cudaError_t launch_xxh64_stream(Xxh64State* st, int op, uint64_t seed, const uint8_t* data, size_t len, cudaStream_t s)
{
    xxh64_stream_kernel<<<1, 32, 0, s>>>(st, op, seed, data, len);
    return cudaGetLastError();
}
#endif

} // namespace b200
