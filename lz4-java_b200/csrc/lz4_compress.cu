// lz4_compress.cu — batch LZ4 fast block compression: launch dispatch and the kernel for blocks above 64 KiB.
//
// Replaces the reference's LZ4_compress_default (lz4.c:1435 -> 1416 -> 1346 -> 910-1302) as called from the JNI shim
// (src/jni/net_jpountz_lz4_LZ4JNI.c:75).  Same algorithm family — greedy single-probe LZ77 over a 4-byte multiplicative
// hash (lz4.c:756-762), 16-bit block-relative positions for blocks < 64 KiB (lz4.c:1353) and 32-bit ones above,
// MFLIMIT/LASTLITERALS end rules (lz4.c:243-244) — re-shaped for 32 lanes, so the emitted stream is a *different valid
// parse* of the same format (like the reference's own Java ports, README.md:45-47): it round-trips bit-exactly through
// every LZ4 decoder; its ratio is reported next to the reference's.
//
//   blocks <= 64 KiB (the bench shape, LZ4Factory.fastCompressor() on 64 KiB blocks): lz4_compress_wide.cuh — three
//       specialised warps per block, 8192 x u16 table;
//   larger blocks (frame blocks up to 4 MiB): lz4_compress_long_kernel below — one warp per block, 4096 x u32 table
//       (the reference's byU32 table, lz4.c:1356).
//
// Algorithmic HBM bytes per block: N (input read once) + C (output written once); tables live in shared memory.
//
// History (DESIGN.md §4): a coupled one-warp parser (41.6 GiB/s), an input-staging variant by TMA (15), the decoupled
// one-warp parser kept below for long blocks (60.5 on 64 KiB blocks), a two-warp pipeline with speculative measurement of
// every hit (89.7), and a three-kernel split through a global arena (37.7) were measured in round 1 and the first half of
// round 2; the shapes that lost are no longer in the library.
#include "common.cuh"
#include "kernels.h"
#include "lz4_emit.cuh"
#include "lz4_compress_wide.cuh"
#include <type_traits>
#include <algorithm>

// Warps per block of the <= 64 KiB kernel: 3 = lookup / parse / layout (the default, measured fastest on the bench corpus),
// 2 = the parser warp also lays out.  A build-time choice (tools/build_variants.sh), not a runtime switch.
#ifndef B200_WIDE_WARPS
#define B200_WIDE_WARPS 3
#endif
// (The tag width of that kernel, B200_WIDE_TAG_BITS, is set in lz4_compress_wide.cuh.)

namespace b200 {

// ---------------------------------------------------------------------------------------------
// One warp per block, any block size (the path for blocks above 64 KiB): candidate lookup + verification run AHEAD of
// the greedy parse.
//
// The coupled kernel above discovers one match, extends it, writes it, and only then knows where to
// probe next: three dependent L2 round trips and ~200 warp instructions per ~27 input bytes, with 13
// warps/SM to hide them.  Here the block is walked in chunks of 128 positions, each in two phases:
//
//   AB (lane-parallel, no decisions): lane l owns the 4 consecutive positions of one aligned 32-bit
//      word of the input (two coalesced word loads + three funnel shifts give its four 4-byte
//      sequences).  All 128 positions are hashed, looked up and then INSERTED (every position, in
//      order), all candidates are verified with four independent loads per lane, and the outcome is
//      one 16-bit distance per position in shared memory (256 B per warp) plus a 128-bit hit mask in
//      registers.  Nothing here depends on the parse.
//   C  (serial, cheap): the greedy walk reads only that: next hit at or after ip from the mask
//      (a few uniform ALU ops), its distance by one shared-memory read, ONE cooperative compare round
//      for catch-up (lz4.c:1080) + the first 24 match bytes (lz4.c:1153), literal copy, and a record
//      of the sequence in lane k's registers.  Tokens and offsets of 32 recorded sequences are then
//      written by 32 lanes at once.
//
// Inserting every position (instead of only positions outside matches) costs no ratio: on the
// reference's own generator the parse is slightly denser than lz4's (1.63 vs 1.61 at P=0.50).
template <int HASH_LOG, bool U16>
__global__ void __launch_bounds__(32)
lz4_compress_long_kernel(const uint8_t* __restrict__ src_base, const uint64_t* __restrict__ src_off,
                          const int32_t* __restrict__ src_len,
                          uint8_t* __restrict__ dst_base, const uint64_t* __restrict__ dst_off,
                          const int32_t* __restrict__ dst_cap, int32_t* __restrict__ result, uint32_t nblocks)
{
    using Entry = typename std::conditional<U16, uint16_t, uint32_t>::type;
    constexpr int TABLE_BYTES = int(sizeof(Entry) << HASH_LOG);
    B200_DYN_SMEM(smem_raw, 128);
    Entry* table = reinterpret_cast<Entry*>(smem_raw);
    uint16_t* s_dist = reinterpret_cast<uint16_t*>(smem_raw + TABLE_BYTES);        // [128] match distance, 0 = no match at this position

    const uint32_t b = blockIdx.x;
    if (b >= nblocks) return;
    const int lane = lane_id();
    const uint8_t* __restrict__ src = src_base + src_off[b];
    uint8_t* __restrict__ dst = dst_base + dst_off[b];
    const int n = src_len[b];
    const int cap = dst_cap[b];
    int ret = 0;

    if (n < 0 || n > 0x7E000000 || cap < 0) goto done;            // lz4.c:1324; no room at all
    if (U16 && n >= 65536 + 11) goto done;                         // lz4.c:973
    if (n == 0) { if (cap >= 1) { if (lane == 0) dst[0] = 0; ret = 1; } goto done; }
    {
        for (int i = lane; i < TABLE_BYTES / 16; i += 32) reinterpret_cast<uint4*>(table)[i] = make_uint4(0, 0, 0, 0);
        __syncwarp();
        // aligned-word view of the block: byte a of the view is position a - ph
        const uint32_t ph = uint32_t(reinterpret_cast<uintptr_t>(src)) & 3u;
        const uint32_t* __restrict__ wsrc = reinterpret_cast<const uint32_t*>(reinterpret_cast<uintptr_t>(src) - ph);
        auto ld4 = [&](int pos) -> uint32_t {                      // the 4 bytes at position pos (pos + 3 < n)
            const uint32_t a = uint32_t(pos) + ph;
            const uint32_t* w = wsrc + (a >> 2);
            return __funnelshift_r(w[0], w[1], (a & 3u) * 8u);
        };
        const int mflimit = n - 12, matchlimit = n - 5;            // lz4.c:243-244
        int op = 0, anchor = 0, ip = 0;
        // up to 32 found sequences wait in registers (lane k holds sequence k) for their token/offset bytes
        int nrec = 0, r_o = 0, r_lit = 0, r_ml = 0, r_dist = 0;

        auto flush = [&]() {                                       // 32 lanes write 32 tokens / length chains / offsets
            if (lane < nrec) {
                const int mcode = r_ml - 4;
                uint8_t* d = dst + r_o;
                d[0] = uint8_t((min(r_lit, 15) << 4) | min(mcode, 15));
                d += 1;
                if (r_lit >= 15) { int v = r_lit - 15; for (; v >= 255; v -= 255) *d++ = 255; *d++ = uint8_t(v); }
                d += r_lit;
                d[0] = uint8_t(r_dist); d[1] = uint8_t(r_dist >> 8);                  // LE16 offset (lz4.c:1133)
                d += 2;
                if (mcode >= 15) { int v = mcode - 15; for (; v >= 255; v -= 255) *d++ = 255; *d++ = uint8_t(v); }
            }
            nrec = 0;
        };

        const int nchunks = (mflimit + int(ph)) / 128 + 1;
        for (int c = 0; c < nchunks; c++) {
            const int cp0 = 128 * c - int(ph);                     // position of the chunk's first byte
            if (lane < 2) {                                        // two chunks ahead -> L2
                const int pfq = cp0 + 512 + lane * 128;
                if (pfq < n) B200_PREFETCH_L2(src + pfq);
            }
            // ---------------- phase AB
            const int p0 = cp0 + 4 * lane;
            uint32_t w0 = 0, w1 = 0;
            if (p0 + 3 >= 0 && p0 <= mflimit) { w0 = wsrc[32 * c + lane]; w1 = wsrc[32 * c + lane + 1]; }
            uint32_t seq[4], h[4]; int cand[4]; bool plaus[4];
            seq[0] = w0; seq[1] = __funnelshift_r(w0, w1, 8); seq[2] = __funnelshift_r(w0, w1, 16); seq[3] = __funnelshift_r(w0, w1, 24);
            #pragma unroll
            for (int j = 0; j < 4; j++) { h[j] = (seq[j] * 2654435761u) >> (32 - HASH_LOG); cand[j] = table[h[j]]; }
            __syncwarp();      // every lookup of the chunk precedes every insert.  Lanes whose sequences hash alike then
                               // store to the same slot: any winner is a valid (earlier) position, so the race is benign
            #pragma unroll
            for (int j = 0; j < 4; j++) {
                const int p = p0 + j;
                const bool valid = p >= 0 && p <= mflimit;
                if (valid) table[h[j]] = Entry(p);
                plaus[j] = valid && cand[j] < p && (U16 || p - cand[j] <= 65535);
            }
            uint32_t cseq[4];
            #pragma unroll
            for (int j = 0; j < 4; j++) cseq[j] = plaus[j] ? ld4(cand[j]) : ~seq[j];
            uint32_t nib = 0; uint32_t d01, d23;
            {
                uint32_t dd[4];
                #pragma unroll
                for (int j = 0; j < 4; j++) {
                    const bool hit = cseq[j] == seq[j];            // implies plaus (otherwise cseq = ~seq)
                    dd[j] = hit ? uint32_t(p0 + j - cand[j]) : 0u;
                    nib |= uint32_t(hit) << j;
                }
                d01 = dd[0] | (dd[1] << 16); d23 = dd[2] | (dd[3] << 16);
            }
            reinterpret_cast<uint2*>(s_dist)[lane] = make_uint2(d01, d23);
            // position-ordered hit mask: word k = positions cp0+32k .. +31 (8 lanes x 4 bits)
            uint32_t gw = nib << (4 * (lane & 7));            // OR over each group of 8 lanes (butterfly: all lanes in step)
            gw |= __shfl_xor_sync(B200_FULL, gw, 1); gw |= __shfl_xor_sync(B200_FULL, gw, 2); gw |= __shfl_xor_sync(B200_FULL, gw, 4);
            const uint32_t hw0 = __shfl_sync(B200_FULL, gw, 0), hw1 = __shfl_sync(B200_FULL, gw, 8),
                           hw2 = __shfl_sync(B200_FULL, gw, 16), hw3 = __shfl_sync(B200_FULL, gw, 24);
            const unsigned long long hlo = (unsigned long long)hw0 | ((unsigned long long)hw1 << 32);
            const unsigned long long hhi = (unsigned long long)hw2 | ((unsigned long long)hw3 << 32);
            __syncwarp();
            // ---------------- phase C: greedy walk over this chunk's hits
            for (;;) {
                int r = ip - cp0;
                if (r < 0) r = 0;
                if (r >= 128) break;
                int q;
                {   // first hit at or after r: two 64-bit halves of the 128-bit position-ordered mask
                    const unsigned long long lo = r < 64 ? (hlo >> r) : 0ull;
                    if (lo) q = r + __ffsll((long long)lo) - 1;
                    else {
                        const int r2 = max(r - 64, 0);
                        const unsigned long long hi = hhi >> r2;
                        if (hi == 0) break;
                        q = 64 + r2 + __ffsll((long long)hi) - 1;
                    }
                }
                int ms = cp0 + q;
                const int dist = s_dist[q];
                int mc = ms - dist, ml;
                {   // one cooperative round: lane j compares offset d = j-8 (catch-up) .. +23 (match body)
                    const int d = lane - 8;
                    const int backroom = min(ms - anchor, mc);
                    const bool ok = d < 0 ? (-d <= backroom) : (ms + d < matchlimit);
                    const bool eq = ok && src[ms + d] == src[mc + d];
                    const unsigned e = __ballot_sync(B200_FULL, eq);
                    const int back = __clz((~e) & 0xFFu) - 24;
                    const int fwd = __ffs((~(e >> 8)) | (1u << 24)) - 1;
                    ml = fwd;
                    if (fwd == 24) ml += match_extend(InGlobal{src}, ms + 24, mc + 24, matchlimit - (ms + 24), lane);
                    ms -= back; ml += back;
                }
                // sizes, literal copy now (offsets are known sequentially), header bytes later in batch
                const int lit = ms - anchor, mcode = ml - 4;
                const int lhdr = lit >= 15 ? (lit - 15) / 255 + 1 : 0;
                const int mhdr = mcode >= 15 ? (mcode - 15) / 255 + 1 : 0;
                const int size = 1 + lhdr + lit + 2 + mhdr;
                if (uint32_t(op) + uint32_t(size) > uint32_t(cap)) goto done;         // lz4.c:1085-1088, 1158 (op <= cap < 2^31)
                warp_copy(dst + op + 1 + lhdr, src + anchor, lit, lane);
                if (lane == nrec) { r_o = op; r_lit = lit; r_ml = ml; r_dist = dist; }
                nrec++;
                if (nrec == 32) flush();
                op += size;
                ip = anchor = ms + ml;
            }
        }
        flush();
        {   // last literals (lz4.c:1266-1293)
            const int lit = n - anchor;
            const int lhdr = lit >= 15 ? (lit - 15) / 255 + 1 : 0;
            if ((long long)op + 1 + lhdr + lit > cap) goto done;
            if (lane == 0) dst[op] = uint8_t(min(lit, 15) << 4);
            op += 1;
            if (lhdr) { write_len_ext(dst + op, lit - 15, lhdr, lane); op += lhdr; }
            warp_copy(dst + op, src + anchor, lit, lane);
            op += lit;
        }
        ret = op;
    }
done:
    if (lane == 0) result[b] = ret;
}

#ifndef B200_HOST_SIM
template <int HASH_LOG, bool U16>
static cudaError_t launch_long(const BatchArgs& a, cudaStream_t st)
{
    const size_t smem = ((U16 ? 2u : 4u) << HASH_LOG) + 128 * sizeof(uint16_t);
    auto k = lz4_compress_long_kernel<HASH_LOG, U16>;
    cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    cudaFuncSetAttribute(k, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    k<<<(unsigned)a.n, 32, smem, st>>>(a.src_base, a.src_off, a.src_len, a.dst_base, a.dst_off, a.dst_cap,
                                       a.result, (uint32_t)a.n);
    return cudaGetLastError();
}
#endif


#ifndef B200_HOST_SIM
#ifdef B200_WIDE_TRACE
// -DB200_WIDE_TRACE builds only: the per-role cycle counts of the last launch (lz4_compress_wide.cuh), first `rows` rows,
// and the CTAs per SM the runtime reports for the kernel that launch used
static int g_wide_ctas_per_sm = 0;
extern "C" int b200lz4_wide_trace_read(unsigned long long* host, int rows)
{
    if (rows < 0 || rows > WIDE_TRACE_ROWS) return -1;
    return cudaMemcpyFromSymbol(host, g_wide_trace, size_t(rows) * WT_N * sizeof(unsigned long long)) == cudaSuccess ? WT_N : -1;
}
extern "C" int b200lz4_wide_trace_ctas_per_sm() { return g_wide_ctas_per_sm; }
#endif

template <int HASH_LOG, int NB, int NW, int TAG_BITS>
static cudaError_t launch_wide(const BatchArgs& a, cudaStream_t st)
{
    constexpr int S = 2;                                                     // sub-rounds of 128 positions per chunk
    using LY = WideLayout<S, NB, NW, TAG_BITS>;
    const size_t smem = LY::smem(HASH_LOG);
    constexpr int FIT = 233472 / (int(LY::smem(HASH_LOG)) + 1024);          // CTAs per SM that shared memory allows
    constexpr int MINB = FIT < 16 ? FIT : 16;
    auto k = lz4_compress_wide_kernel<HASH_LOG, S, NB, NW, MINB, TAG_BITS>;
    cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    cudaFuncSetAttribute(k, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
#ifdef B200_WIDE_TRACE
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&g_wide_ctas_per_sm, k, 32 * NW, smem);
#endif
    k<<<(unsigned)a.n, 32 * NW, smem, st>>>(a.src_base, a.src_off, a.src_len, a.dst_base, a.dst_off, a.dst_cap, a.result, (uint32_t)a.n);
    return cudaGetLastError();
}


cudaError_t launch_compress_fast(const BatchArgs& a, int max_src_len, cudaStream_t st)
{
    if (a.n == 0) return cudaSuccess;
    if (max_src_len > 0 && max_src_len <= 65536) return launch_wide<13, 2, B200_WIDE_WARPS, B200_WIDE_TAG_BITS>(a, st);   // 8192 x u16: lz4.c:1353
    return launch_long<12, false>(a, st);                  // 4096 x u32 = 16 KiB, the reference's byU32 table (lz4.c:1356)
}
#endif

} // namespace b200
