// lz4_compress_wide.cuh — fast LZ4 block compression for blocks < 64 KiB (algo 5): a lookup warp that verifies 8 bytes per
// candidate and a parser warp that walks the greedy chain on shared-memory state alone.
//
// Replaces the reference's LZ4_compress_default for byU16 blocks (lz4.c:1435 -> 1346 -> 910-1302, called from
// src/jni/net_jpountz_lz4_LZ4JNI.c:75).  Same algorithm family: greedy single-probe LZ77 over the 4-byte multiplicative
// hash (lz4.c:756-762), 8192 x u16 block-relative positions (lz4.c:1353), catch-up (lz4.c:1080), MFLIMIT / LASTLITERALS
// end rules (lz4.c:243-244).  Every position is probed AND inserted, so the stream is a different valid parse of the same
// format (ratio next to the reference's in bench.py); it is byte-identical to what lz4_compress_fast3_kernel emits.
//
// Why this shape (round-2 measurements, tools/study/fast_parse_study.c): on the bench corpus 512 input bytes hold ~114
// hits in ~68 runs but only ~20 selected sequences, and 82 % of the selected matches are shorter than 8 bytes.  Measuring
// hits speculatively (the round-1 parser: 14 loads per hit, 32 hits per round) spends most of its instructions on hits the
// greedy chain then skips.  Here
//   warp L  walks the block in chunks of 128*S positions, S sub-rounds of 128 in order: probe 4 positions per lane,
//           barrier, insert, then verify every candidate whose hash tag matches (TAG_BITS below) against EIGHT bytes (three
//           aligned words of the position, one aligned 16-byte load of the candidate, two when they straddle it).  Per position
//           it publishes a u16 distance and a byte: the verified length (4..8) and how far the next hit behind the match is; per
//           chunk a hit mask.
//   warp P  walks the chain on warp-uniform values: two shared-memory loads per sequence give distance, length and the
//           position of the next sequence.  Only a match whose 8 verified bytes all agreed is extended, cooperatively (128
//           bytes per round), and only then (or when the next hit is more than 32 positions away) is the hit mask searched.  Lane k keeps sequence k; every 32 sequences the warp lays them out at once: catch-up for 32 sequences
//           in one batch of loads, prefix sum of sizes, token / length bytes / offset, lane-parallel literal copies.
//   warp E  (three-warp build, NW = 3) takes the layout off warp P: P writes 8-byte records into shared memory, E lays out
//           batches of 32 while P walks on.
// Hand-off: named barriers per chunk buffer (L: bar.arrive FULL, P: bar.sync FULL ... bar.arrive FREE), NB buffers; one more
// pair for the record batch.
//
// Algorithmic HBM bytes per block: N (input, read once) + C (output, written once); table and chunk state live in
// shared memory.
#pragma once
#include "common.cuh"
#include "lz4_emit.cuh"
#include <type_traits>

// Hash-tag bits per table slot (0, 1, 2, 4 or 8; 0 = no tags), the default of the kernel's TAG_BITS.  Every width emits the
// same bytes; wider tags skip more verify loads but leave room for fewer CTAs per SM (shared memory: 12, 11, 10, 9, 8; the
// runtime reports 9 for the untagged kernel).  8 measured fastest on the bench corpus (DESIGN.md §4).  A build-time choice
// (tools/build_variants.sh), not a runtime switch.
#ifndef B200_WIDE_TAG_BITS
#define B200_WIDE_TAG_BITS 8
#endif

namespace b200 {

#ifdef B200_HOST_SIM
__device__ __forceinline__ void wide_bar_arrive(int id) { simt::bar_arrive(id, 64); }
__device__ __forceinline__ void wide_bar_wait(int id) { simt::bar_sync(id, 64); }
__device__ __forceinline__ uint32_t ldg_u32(const uint32_t* p) { return *p; }
__device__ __forceinline__ void ldg_pair(const uint32_t* base, uint32_t idx, uint32_t& lo, uint32_t& hi) { lo = base[idx]; hi = base[idx + 1]; }
__device__ __forceinline__ uint4 ldg_u128(const uint4* p) { return *p; }
__device__ __forceinline__ void shared_xor(uint32_t* p, uint32_t v) { *p ^= v; }     // (the emulator runs one lane at a time)
#else
// (Immediate barrier ids, so ptxas reserves only the barriers in use and not all 16.)
#define B200_WBAR_CASE(OP, N) case N: asm volatile(OP " " #N ", 64;" ::: "memory"); break;
__device__ __forceinline__ void wide_bar_arrive(int id)
{
    switch (id) { B200_WBAR_CASE("bar.arrive", 1) B200_WBAR_CASE("bar.arrive", 2) B200_WBAR_CASE("bar.arrive", 3)
                  B200_WBAR_CASE("bar.arrive", 4) B200_WBAR_CASE("bar.arrive", 5) default: asm volatile("bar.arrive 6, 64;" ::: "memory"); }
}
__device__ __forceinline__ void wide_bar_wait(int id)
{
    switch (id) { B200_WBAR_CASE("bar.sync", 1) B200_WBAR_CASE("bar.sync", 2) B200_WBAR_CASE("bar.sync", 3)
                  B200_WBAR_CASE("bar.sync", 4) B200_WBAR_CASE("bar.sync", 5) default: asm volatile("bar.sync 6, 64;" ::: "memory"); }
}
__device__ __forceinline__ uint32_t ldg_u32(const uint32_t* p) { return __ldg(p); }      // the input is read-only for the kernel
__device__ __forceinline__ uint4 ldg_u128(const uint4* p) { return __ldg(p); }
__device__ __forceinline__ void shared_xor(uint32_t* p, uint32_t v) { atomicXor(p, v); }
// words idx and idx + 1 of a read-only array: one 32x32+64 multiply-add for the address, two loads off it
__device__ __forceinline__ void ldg_pair(const uint32_t* base, uint32_t idx, uint32_t& lo, uint32_t& hi)
{
    uint64_t a;
    asm("mad.wide.u32 %0, %1, 4, %2;" : "=l"(a) : "r"(idx), "l"(base));
    asm("ld.global.nc.u32 %0, [%1];" : "=r"(lo) : "l"(a));
    asm("ld.global.nc.u32 %0, [%1+4];" : "=r"(hi) : "l"(a));
}
#endif

// Per-role cycle accounting (builds with -DB200_WIDE_TRACE only; tools/compress_roles.py reads it): every 64th CTA, lane 0
// of each warp adds up the clock64 cycles its warp spends in the marked waits and calls and writes them, with its total, to
// row blockIdx / 64 of g_wide_trace.  Without the flag the macros are empty and the kernel is the same code.
#ifdef B200_WIDE_TRACE
enum { WT_L_TOTAL, WT_L_FREE, WT_E_TOTAL, WT_E_REC_FULL, WT_P_TOTAL, WT_P_FULL, WT_P_REC_FREE, WT_P_EXTEND, WT_P_SEARCH,
       WT_SEQUENCES, WT_EXTENDS, WT_SEARCHES, WT_N };           // (tools/compress_roles.py reads the rows in this order)
constexpr int WIDE_TRACE_EVERY = 64, WIDE_TRACE_ROWS = 16384;
__device__ unsigned long long g_wide_trace[WIDE_TRACE_ROWS][WT_N];
#define WT_BEGIN unsigned long long wt[WT_N] = {}; const long long wt_start = clock64()
#define WT_TIME(slot, ...) do { const long long t_ = clock64(); __VA_ARGS__; wt[slot] += clock64() - t_; } while (0)
#define WT_COUNT(slot) (wt[slot] += 1)
#define WT_END(total, lo, hi) do {                                                                                   \
        wt[total] = clock64() - wt_start;                                                                           \
        if (lane == 0 && b % WIDE_TRACE_EVERY == 0 && b / WIDE_TRACE_EVERY < WIDE_TRACE_ROWS) {                     \
            g_wide_trace[b / WIDE_TRACE_EVERY][total] = wt[total];                                                 \
            for (int i_ = lo; i_ < hi; i_++) g_wide_trace[b / WIDE_TRACE_EVERY][i_] = wt[i_];                      \
        } } while (0)
#else
#define WT_BEGIN
#define WT_TIME(slot, ...) do { __VA_ARGS__; } while (0)
#define WT_COUNT(slot)
#define WT_END(total, lo, hi)
#endif

template <int S, int NB, int NW, int TAG_BITS>
struct WideLayout {
    static constexpr int CH = 128 * S;                 // positions per chunk
    static constexpr int MW = CH / 32;                 // mask words per chunk
    static constexpr int BUF_BYTES = CH * 3 + MW * 4;  // u16 distances + u8 jump/length codes + hit mask
    static constexpr int REC_BYTES = 32 * 8 + 16;      // one batch of sequence records + its header
    static constexpr size_t tag_bytes(int hash_log) { return (size_t(TAG_BITS) << hash_log) / 8; }
    static constexpr size_t smem(int hash_log)
    { return (size_t(2) << hash_log) + tag_bytes(hash_log) + size_t(NB) * BUF_BYTES + REC_BYTES; }
};

// TAG_BITS > 0: next to every table slot the lookup warp keeps TAG_BITS more bits of the hash of the position stored
// there (the bits of the same product just below the slot index).  A candidate whose tag differs from the probing
// position's own cannot share its first 4 bytes, so its verify loads are not issued.  TAG_BITS = 0 is the plain table.
template <int HASH_LOG, int S, int NB, int NW, int MINB, int TAG_BITS = B200_WIDE_TAG_BITS>
__global__ void __launch_bounds__(32 * NW, MINB)
lz4_compress_wide_kernel(const uint8_t* __restrict__ src_base, const uint64_t* __restrict__ src_off,
                         const int32_t* __restrict__ src_len,
                         uint8_t* __restrict__ dst_base, const uint64_t* __restrict__ dst_off,
                         const int32_t* __restrict__ dst_cap, int32_t* __restrict__ result, uint32_t nblocks)
{
    using LY = WideLayout<S, NB, NW, TAG_BITS>;
    constexpr int CH = LY::CH, MW = LY::MW;
    constexpr int TABLE_BYTES = 2 << HASH_LOG;
    constexpr int TAG_BYTES = int(LY::tag_bytes(HASH_LOG));
    constexpr int BAR_FULL = 1, BAR_FREE = 1 + NB, BAR_REC_FULL = 1 + 2 * NB, BAR_REC_FREE = 2 + 2 * NB;
    constexpr int REC_LAST = 0x100;                        // batch header flag: no batch follows
    static_assert(NW == 2 || NW == 3, "two or three warps");
    static_assert(2 * NB + (NW == 3 ? 2 : 0) <= 6, "named barrier ids 1..6");
    static_assert(TAG_BITS == 0 || TAG_BITS == 1 || TAG_BITS == 2 || TAG_BITS == 4 || TAG_BITS == 8, "tag widths 0, 1, 2, 4, 8");
    B200_DYN_SMEM(smem_raw, 128);
    uint16_t* table = reinterpret_cast<uint16_t*>(smem_raw);
    uint8_t* tags = smem_raw + TABLE_BYTES;               // TAG_BITS per slot, slot h at bit TAG_BITS * h
    uint8_t* bufs = smem_raw + TABLE_BYTES + TAG_BYTES;
    auto dist_of = [&](int buf) { return reinterpret_cast<uint16_t*>(bufs + buf * LY::BUF_BYTES); };
    auto flen_of = [&](int buf) { return bufs + buf * LY::BUF_BYTES + CH * 2; };
    auto hmask_of = [&](int buf) { return reinterpret_cast<uint32_t*>(bufs + buf * LY::BUF_BYTES + CH * 3); };
    uint2* s_rec = reinterpret_cast<uint2*>(bufs + NB * LY::BUF_BYTES);                  // [32] x = start | distance << 16, y = length
    int* s_hdr = reinterpret_cast<int*>(bufs + NB * LY::BUF_BYTES + 256);                // [0] records | REC_LAST, [1] end of the parse

    const uint32_t b = blockIdx.x;
    if (b >= nblocks) return;
    const int lane = lane_id();
    const int role = threadIdx.x >> 5;                     // 0 = L (lookup), 1 = P (parse; + layout when NW == 2), 2 = E (layout)
    const uint8_t* __restrict__ src = src_base + src_off[b];
    uint8_t* __restrict__ dst = dst_base + dst_off[b];
    const int n = src_len[b];
    const int cap = dst_cap[b];

    if (n < 0 || n >= 65536 + 11 || cap < 0) { if (threadIdx.x == 0) result[b] = 0; return; }     // lz4.c:1324, 973; no room at all
    if (n == 0) { if (threadIdx.x == 0) { if (cap >= 1) dst[0] = 0; result[b] = cap >= 1 ? 1 : 0; } return; }   // lz4.c:1325-1336
    WT_BEGIN;

    // aligned-word view of the block: byte a of the view is position a - ph
    const uint32_t ph = uint32_t(reinterpret_cast<uintptr_t>(src)) & 3u;
    const uint32_t* __restrict__ wsrc = reinterpret_cast<const uint32_t*>(reinterpret_cast<uintptr_t>(src) - ph);
    const uint32_t ph16 = uint32_t(reinterpret_cast<uintptr_t>(src)) & 15u;               // ... and the same in 16-byte words
    const uint4* __restrict__ osrc = reinterpret_cast<const uint4*>(reinterpret_cast<uintptr_t>(src) - ph16);
    const int mflimit = n - 12, matchlimit = n - 5;        // lz4.c:243-244
    const int nchunks = mflimit >= 0 ? (mflimit + int(ph)) / CH + 1 : 0;     // n < 13: all literals (lz4.c:981)
    auto ld4 = [&](int pos) -> uint32_t {                  // the 4 bytes at position pos
        const uint32_t a = uint32_t(pos) + ph;
        uint32_t lo, hi;
        ldg_pair(wsrc, a >> 2, lo, hi);
        return __funnelshift_r(lo, hi, a << 3);
    };

    if (role == 0) {
        // ================================================================== warp L: probe, insert, verify 8 bytes
        constexpr uint32_t TMASK = (1u << TAG_BITS) - 1u;
        auto tag_of = [](uint32_t prod) { return (prod >> (32 - HASH_LOG - TAG_BITS)) & TMASK; };
        uint32_t* tagw = reinterpret_cast<uint32_t*>(tags);
        auto tag_get = [&](uint32_t h) { return (tagw[(TAG_BITS * h) >> 5] >> ((TAG_BITS * h) & 31u)) & TMASK; };
        // An untouched slot holds position 0, so its tag starts as position 0's: the probes of the first sub-round run before
        // position 0 is inserted and may still find it (bytes 0..3 == p..p+3 at the start of a run).
        const uint32_t tag0 = (TAG_BITS && nchunks) ? tag_of(ld4(0) * 2654435761u) * (0xFFFFFFFFu / max(TMASK, 1u)) : 0u;
        for (int i = lane; i < TABLE_BYTES / 16; i += 32) reinterpret_cast<uint4*>(table)[i] = make_uint4(0, 0, 0, 0);
        for (int i = lane; i < TAG_BYTES / 16; i += 32) reinterpret_cast<uint4*>(tags)[i] = make_uint4(tag0, tag0, tag0, tag0);
        __syncwarp();
        // One chunk.  EDGE = false is the body for chunks whose positions are all inside [1, mflimit): there every position is
        // valid, every table entry is a position inserted earlier (< p) and 8 bytes fit below matchlimit, so no validity
        // predicate is left in the code.
        auto lookup = [&](int c, auto edge_tag) {
            constexpr bool EDGE = decltype(edge_tag)::value;
            const int buf = c % NB;
            const int cp0 = CH * c - int(ph);
            // ---- phase 1, sub-round by sub-round: probe all 128 positions, then insert all 128
            uint32_t w0[S], w1[S], w2[S]; int cand[S][4];
            uint32_t tok = TAG_BITS ? 0u : 0xFFFFFFFFu;    // bit 4s + j: the candidate's tag equals the position's own
            #pragma unroll
            for (int s = 0; s < S; s++) {
                const int p0 = cp0 + 128 * s + 4 * lane;
                const uint32_t* wp = wsrc + (uint32_t(CH / 4) * uint32_t(c) + 32u * uint32_t(s) + uint32_t(lane));
                w0[s] = w1[s] = w2[s] = 0;
                if (!EDGE || (p0 + 3 >= 0 && p0 <= mflimit)) { w0[s] = ldg_u32(wp); w1[s] = ldg_u32(wp + 1); w2[s] = ldg_u32(wp + 2); }
            }
            #pragma unroll
            for (int s = 0; s < S; s++) {
                const int p0 = cp0 + 128 * s + 4 * lane;
                uint32_t h[4];
                [[maybe_unused]] uint32_t t[4], ct[4];                                           // (TAG_BITS > 0)
                #pragma unroll
                for (int j = 0; j < 4; j++) {
                    const uint32_t sq = j ? __funnelshift_r(w0[s], w1[s], 8 * j) : w0[s];
                    const uint32_t prod = sq * 2654435761u;
                    h[j] = prod >> (32 - HASH_LOG);
                    cand[s][j] = table[h[j]];
                    if constexpr (TAG_BITS > 0) {
                        t[j] = tag_of(prod);
                        ct[j] = tag_get(h[j]);
                        tok |= uint32_t(ct[j] == t[j]) << (4 * s + j);
                    }
                }
                __syncwarp();  // every probe of the sub-round precedes every insert (same-slot stores: any winner is a valid position)
                #pragma unroll
                for (int j = 0; j < 4; j++) {
                    const int p = p0 + j;
                    if (!EDGE || (p >= 0 && p <= mflimit)) table[h[j]] = uint16_t(p);
                }
                __syncwarp();  // ... and every insert precedes the next sub-round's probes
                if constexpr (TAG_BITS > 0) {
                    // Only the lane whose position won the slot writes its tag, so a slot never pairs one lane's position with
                    // another's tag, however the same-slot stores above were ordered.  Nobody else writes those tag bits in this
                    // sub-round, so they still hold ct (what this lane probed): one XOR of ct ^ t sets them, and lanes that share
                    // a word touch disjoint bits.
                    #pragma unroll
                    for (int j = 0; j < 4; j++) {
                        const int p = p0 + j;
                        if ((!EDGE || (p >= 0 && p <= mflimit)) && table[h[j]] == uint16_t(p)) {
                            if constexpr (TAG_BITS == 8) tags[h[j]] = uint8_t(t[j]);
                            else if (ct[j] != t[j]) shared_xor(&tagw[(TAG_BITS * h[j]) >> 5], (ct[j] ^ t[j]) << ((TAG_BITS * h[j]) & 31u));
                        }
                    }
                    __syncwarp();  // every tag is written before the next sub-round's probes
                }
            }
            // ---- phase 2: all candidates of the chunk are verified with independent loads (one L2 round trip per chunk)
            if (c >= NB) WT_TIME(WT_L_FREE, wide_bar_wait(BAR_FREE + buf));    // warp P is done with this buffer's previous tenant
            uint16_t* ds = dist_of(buf);
            uint8_t* fls = flen_of(buf);
            uint32_t* hm = hmask_of(buf);
            uint32_t fl[S][4], gh[S];                      // per sub-round: the lane's four verified lengths, its group's hit word
            #pragma unroll
            for (int s = 0; s < S; s++) {
                const int p0 = cp0 + 128 * s + 4 * lane;
                uint32_t dd[4], nib = 0;
                #pragma unroll
                for (int j = 0; j < 4; j++) {
                    const int p = p0 + j;
                    const uint32_t sq = j ? __funnelshift_r(w0[s], w1[s], 8 * j) : w0[s];        // bytes p .. p+3
                    const uint32_t sn = j ? __funnelshift_r(w1[s], w2[s], 8 * j) : w1[s];        // bytes p+4 .. p+7
                    const bool plaus = (!EDGE || (p >= 0 && p <= mflimit && cand[s][j] < p)) && ((tok >> (4 * s + j)) & 1u);
                    // The candidate's 8 bytes: its aligned 16-byte word, and the next one only when they straddle it.  No
                    // load for an implausible candidate; what is computed from the zeros then is never read (no hit bit).
                    const uint32_t a = uint32_t(cand[s][j]) + ph16;
                    const uint4* w = osrc + (a >> 4);
                    uint4 v = make_uint4(0, 0, 0, 0), v2 = make_uint4(0, 0, 0, 0);
                    if (plaus) v = ldg_u128(w);
                    if (plaus && (a & 15u) > 8u) v2 = ldg_u128(w + 1);
                    const bool h8 = (a & 8u) != 0;                                               // the two aligned 8-byte words
                    const uint2 q0 = h8 ? make_uint2(v.z, v.w) : make_uint2(v.x, v.y);
                    const uint2 q1 = h8 ? make_uint2(v2.x, v2.y) : make_uint2(v.z, v.w);
                    const bool up = (a & 4u) != 0;
                    const uint32_t c0 = up ? q0.y : q0.x, c1 = up ? q1.x : q0.y, c2 = up ? q1.y : q1.x;
                    const uint32_t x = __funnelshift_r(c0, c1, a << 3) ^ sq;
                    const uint32_t y = __funnelshift_r(c1, c2, a << 3) ^ sn;
                    dd[j] = EDGE ? (uint32_t(p - cand[s][j]) & 0xFFFFu) : uint32_t(p - cand[s][j]);
                    fl[s][j] = 4u + min((uint32_t(__ffs(int(y))) - 1u) >> 3, 4u);                // 4 + equal bytes among p+4 .. p+7 (__ffs(0) = 0)
                    if (EDGE) fl[s][j] = uint32_t(min(int(fl[s][j]), max(matchlimit - p, 4)));   // matches end at matchlimit (lz4.c:943)
                    nib |= uint32_t(plaus && x == 0) << j;
                }
                reinterpret_cast<uint2*>(ds + 128 * s)[lane] = make_uint2(dd[0] | (dd[1] << 16), dd[2] | (dd[3] << 16));
                // position-ordered hit mask: word k of the sub-round = positions 32k .. 32k+31 (8 lanes x 4 bits)
                uint32_t g = nib << (4u * (uint32_t(lane) & 7u));
                g |= __shfl_xor_sync(B200_FULL, g, 1); g |= __shfl_xor_sync(B200_FULL, g, 2); g |= __shfl_xor_sync(B200_FULL, g, 4);
                if ((lane & 7) == 0) hm[4 * s + (lane >> 3)] = g;
                gh[s] = g;
            }
            // ---- the chain's jump table: for a hit at p with verified length fl < 8 the parser needs the first hit at or after
            // p + fl.  Every lane looks it up in the 32 positions behind p0 + 4 (its own group's word and the next one; past the end
            // of the chunk there is nothing, the parser searches the next chunk itself).  Byte per position:
            //   (fl - 4) << 6 | distance to that hit (0 = none among the 32),   0xFF = all 8 bytes agreed, length still open.
            #pragma unroll
            for (int s = 0; s < S; s++) {
                uint32_t nx = __shfl_down_sync(B200_FULL, gh[s], 8);                               // the next group's word
                const uint32_t nxs = (s + 1 < S) ? __shfl_sync(B200_FULL, gh[(s + 1) % S], 0) : 0u;   // first word of the next sub-round
                if (lane >= 24) nx = nxs;
                const uint32_t win = __funnelshift_rc(gh[s], nx, 4u * (uint32_t(lane) & 7u) + 4u);    // hits at p0+4 .. p0+35
                uint32_t out = 0;
                #pragma unroll
                for (int j = 0; j < 4; j++) {
                    const uint32_t f = fl[s][j];
                    const uint32_t mm = win >> (uint32_t(j) + f - 4u);                                // hits at p + f ..
                    const uint32_t z = uint32_t(__ffs(int(mm))) - 1u;                                 // 0xFFFFFFFF when there is none
                    const uint32_t code = min(f * 64u - 256u + (z < 32u ? f + z : 0u), 0xFFu);        // f == 8 -> 0xFF
                    out |= code << (8 * j);
                }
                reinterpret_cast<uint32_t*>(fls + 128 * s)[lane] = out;
            }
            wide_bar_arrive(BAR_FULL + buf);
        };
        for (int c = 0; c < nchunks; c++) {
            const int cp0 = CH * c - int(ph);
            if (lane < S) {                                // two chunks ahead -> L2
                const int pfq = cp0 + 2 * CH + lane * 128;
                if (pfq < n) B200_PREFETCH_L2(src + pfq);
            }
            if (c > 0 && cp0 + CH - 1 < mflimit) lookup(c, std::false_type{});
            else lookup(c, std::true_type{});
        }
        WT_END(WT_L_TOTAL, WT_L_FREE, WT_L_FREE + 1);
        return;
    }

    // ====================================================================== warps P and E
    int ip = 0;                                            // end of the last selected match = start of the pending literals
    int op = 0; bool fail = false;
    int k = 0;                                             // sequences waiting: in registers (lane j holds sequence j) or in s_rec
    int r_pend = 0, r_ms = 0, r_len = 4, r_dist = 1;

    // equal bytes between positions a.. and (a - dist).., at most maxlen (>= 0): 4 bytes per lane, 128 per round
    auto extend = [&](int a, int dist, int maxlen) -> int {
        int total = 0;
        for (;;) {
            const int i = total + 4 * lane;
            uint32_t x = 1;                                    // "differs at byte 0" beyond the limit
            if (i < maxlen) x = ld4(a + i) ^ ld4(a + i - dist);
            const unsigned neq = __ballot_sync(B200_FULL, x != 0);
            if (neq) {
                const int fl = __ffs(neq) - 1;
                const uint32_t xf = __shfl_sync(B200_FULL, x, fl);
                return min(total + 4 * fl + ((__ffs(xf) - 1) >> 3), maxlen);
            }
            total += 128;
        }
    };

    // lay out cnt sequences, lane j holds sequence j (lz4.c:1080, 1094-1100, 1133, 1184-1196)
    auto layout = [&](int cnt) {
        const bool on = lane < cnt;
        int start = r_ms, len = r_len;
        if (on && r_ms - r_dist >= 4 && r_ms > r_pend) {      // catch-up: up to 4 equal bytes behind the match (lz4.c:1080)
            const uint32_t x = ld4(r_ms - 4) ^ ld4(r_ms - r_dist - 4);
            const int back = x ? (__clz(x) >> 3) : 4;
            const int bk = min(back, r_ms - r_pend);
            start -= bk; len += bk;
        }
        const int lit = on ? start - r_pend : 0, mcode = len - 4;
        const int lhdr = lit >= 15 ? (lit - 15) / 255 + 1 : 0;
        const int mhdr = (on && mcode >= 15) ? (mcode - 15) / 255 + 1 : 0;
        const int size = on ? 1 + lhdr + lit + 2 + mhdr : 0;
        int incl = size;
        #pragma unroll
        for (int d = 1; d < 32; d <<= 1) { const int y = __shfl_up_sync(B200_FULL, incl, d); if (lane >= d) incl += y; }
        const int total = __shfl_sync(B200_FULL, incl, 31);
        if (fail) return;
        if (uint32_t(op) + uint32_t(total) > uint32_t(cap)) { fail = true; return; }               // lz4.c:1085-1088, 1158
        const int o = op + incl - size;
        if (on) {
            uint8_t* d = dst + o;
            d[0] = uint8_t((min(lit, 15) << 4) | min(mcode, 15));
            d += 1;
            if (lit >= 15) { int v = lit - 15; for (; v >= 255; v -= 255) *d++ = 255; *d++ = uint8_t(v); }
            d += lit;
            d[0] = uint8_t(r_dist); d[1] = uint8_t(r_dist >> 8);                                 // LE16 offset (lz4.c:1133)
            d += 2;
            if (mcode >= 15) { int v = mcode - 15; for (; v >= 255; v -= 255) *d++ = 255; *d++ = uint8_t(v); }
        }
        // Literal runs: every lane copies the first 32 bytes of its own run (the runs of one batch lie within a few lines
        // of each other, so the 32 lanes' byte accesses coalesce); the longer runs are finished by the whole warp.
        uint8_t* lo = dst + o + 1 + lhdr;
        const int sn = min(lit, 32);
        const int mx = __reduce_max_sync(B200_FULL, sn);
        for (int t = 0; t < mx; t += 4) {
            if (t < sn) {
                const uint32_t v = ld4(r_pend + t);
                lo[t] = uint8_t(v);
                if (t + 1 < sn) lo[t + 1] = uint8_t(v >> 8);
                if (t + 2 < sn) lo[t + 2] = uint8_t(v >> 16);
                if (t + 3 < sn) lo[t + 3] = uint8_t(v >> 24);
            }
        }
        for (unsigned lm = __ballot_sync(B200_FULL, lit > 32); lm; lm &= lm - 1) {
            const int j = __ffs(lm) - 1;
            const int ka = __shfl_sync(B200_FULL, r_pend, j);
            const int kl = __shfl_sync(B200_FULL, lit, j);
            const int ko = __shfl_sync(B200_FULL, o + 1 + lhdr, j);
            warp_copy(dst + ko + 32, src + ka + 32, kl - 32, lane);
        }
        op += total;
    };

    auto finish = [&](int fin) {                           // last literals (lz4.c:1266-1293)
        int ret = 0;
        if (!fail) {
            const int lit = n - fin;
            const int lhdr = lit >= 15 ? (lit - 15) / 255 + 1 : 0;
            if (uint32_t(op) + 1u + uint32_t(lhdr) + uint32_t(lit) <= uint32_t(cap)) {
                if (lane == 0) dst[op] = uint8_t(min(lit, 15) << 4);
                op += 1;
                if (lhdr) { write_len_ext(dst + op, lit - 15, lhdr, lane); op += lhdr; }
                warp_copy(dst + op, src + fin, lit, lane);
                ret = op + lit;
            }
        }
        if (lane == 0) result[b] = ret;
    };

    // lay out the batch in s_rec: lane j takes sequence j; prev_end = end of the sequence before the batch
    int prev_end = 0;
    auto layout_batch = [&](int cnt) {
        uint2 r = make_uint2(0, 4);
        if (lane < cnt) r = s_rec[lane];
        if (NW == 3) wide_bar_arrive(BAR_REC_FREE);                    // the batch is in registers: warp P may write the next one
        r_ms = int(r.x & 0xFFFFu); r_dist = int(r.x >> 16); r_len = int(r.y);
        const int end = r_ms + r_len;
        r_pend = __shfl_up_sync(B200_FULL, end, 1);
        if (lane == 0) r_pend = prev_end;
        if (cnt > 0) prev_end = __shfl_sync(B200_FULL, end, cnt - 1);
        layout(cnt);
    };

    if (NW == 3 && role == 2) {
        // ================================================================== warp E: lay out batches of 32 sequences
        for (;;) {
            WT_TIME(WT_E_REC_FULL, wide_bar_wait(BAR_REC_FULL));
            const int hdr = s_hdr[0], fin = s_hdr[1];
            layout_batch(hdr & 0xFF);
            if (hdr & REC_LAST) { finish(fin); break; }
        }
        WT_END(WT_E_TOTAL, WT_E_REC_FULL, WT_E_REC_FULL + 1);
        return;
    }

    // ================================================================== warp P: the greedy chain
    auto flush = [&](bool last) {
        if (NW == 2) { __syncwarp(); layout_batch(k); k = 0; __syncwarp(); return; }
        if (lane == 0) { s_hdr[0] = k | (last ? REC_LAST : 0); s_hdr[1] = ip; }
        wide_bar_arrive(BAR_REC_FULL);
        WT_TIME(WT_P_REC_FREE, wide_bar_wait(BAR_REC_FREE));    // warp E has the batch in registers (it answers at once)
        k = 0;
    };
    for (int c = 0; c < nchunks; c++) {
        const int buf = c % NB;
        const int cp0 = CH * c - int(ph);
        WT_TIME(WT_P_FULL, wide_bar_wait(BAR_FULL + buf));
        const uint16_t* ds = dist_of(buf);
        const uint8_t* fls = flen_of(buf);
        const uint32_t* hm = hmask_of(buf);
        // first hit at or after chunk position r (warp-uniform), CH if there is none
        auto search = [&](uint32_t r) -> uint32_t {
            if (r >= uint32_t(CH)) return CH;
            uint32_t w = r >> 5;
            uint32_t m = hm[w] & (0xFFFFFFFFu << (r & 31u));
            while (m == 0 && ++w < uint32_t(MW)) m = hm[w];
            return m ? 32u * w + uint32_t(__ffs(int(m))) - 1u : uint32_t(CH);
        };
        uint32_t q;
        WT_TIME(WT_P_SEARCH, q = search(uint32_t(max(ip - cp0, 0)))); WT_COUNT(WT_SEARCHES);
        uint32_t code = 0, dist = 0;
        if (q < uint32_t(CH)) { code = fls[q]; dist = ds[q]; }
        while (q < uint32_t(CH)) {
            const uint32_t ms = uint32_t(cp0) + q;
            uint32_t fl = 4u + (code >> 6);
            const uint32_t delta = code & 63u;
            uint32_t nq = q + delta;
            if (delta - 1u >= 62u) {                          // rare: the length is still open (63) or no hit among the next 32 positions (0)
                if (delta) { WT_TIME(WT_P_EXTEND, fl = 8u + uint32_t(extend(int(ms) + 8, int(dist), matchlimit - (int(ms) + 8)))); WT_COUNT(WT_EXTENDS); }
                WT_TIME(WT_P_SEARCH, nq = search(q + fl)); WT_COUNT(WT_SEARCHES);
            }
            // the next sequence's two loads go out before this one is booked: their latency is the chain's critical path
            // (unconditionally: nq is at most 62 entries past the chunk, still inside this CTA's shared memory, and a value
            // read there is never used -- the loop ends)
            const uint32_t ncode = fls[nq], ndist = ds[nq];
            if (lane == 0) s_rec[k] = make_uint2(ms | (dist << 16), fl);
            ip = int(ms + fl);
            q = nq; code = ncode; dist = ndist;
            WT_COUNT(WT_SEQUENCES);
            if (++k == 32) flush(false);
        }
        if (c + NB < nchunks) wide_bar_arrive(BAR_FREE + buf);
    }
    flush(true);
    if (NW == 2) finish(ip);
    WT_END(WT_P_TOTAL, WT_P_FULL, WT_N);
}

} // namespace b200
