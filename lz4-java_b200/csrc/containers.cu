// containers.cu — the containers lz4-java wraps around the block codec, as whole-buffer batch calls:
//   * LZ4 Frame writer     — LZ4FrameOutputStream.writeHeader/writeBlock/writeEndMark
//                            (src/java/net/jpountz/lz4/LZ4FrameOutputStream.java:178-251)
//   * "LZ4Block" container — LZ4BlockOutputStream.flushBufferedData/finish (:203-266) and
//                            LZ4BlockInputStream.refill (LZ4BlockInputStream.java:191-264)
//   * length-prefixed block — LZ4CompressorWithLength / LZ4DecompressorWithLength
// The reference does these one block per native call.  Here the frame is written on the device (frame_encode.cu), and the
// LZ4Block container's host code only lays out headers while the payload work (block compression / decompression, every
// XXH32) goes through the batch entry points, i.e. the CUDA kernels.  No hashing or codec arithmetic runs on the host.
#include "../../include/b200lz4.h"
#include "kernels.h"
#ifdef B200_HOST_SIM            // the emulator build compiles the host layer only: the device frame writer's kernels come with it
#include "frame_encode.cu"
#endif
#include <cstdlib>
#include <cstring>
#include <vector>

static inline void put32(uint8_t* p, uint32_t v) { p[0] = (uint8_t)v; p[1] = (uint8_t)(v >> 8); p[2] = (uint8_t)(v >> 16); p[3] = (uint8_t)(v >> 24); }
static inline uint32_t get32(const uint8_t* p) { return p[0] | (p[1] << 8) | (p[2] << 16) | ((uint32_t)p[3] << 24); }

// The LZ4Block writer's compressor argument (LZ4BlockOutputStream takes any LZ4Compressor): hc_level 0 = the fast
// compressor, packed output; 1..17 = LZ4_compress_HC at that level into bound-sized slots.  coff/clen as *_compact_host.
static int compress_blocks(const uint8_t* src, const uint64_t* soff, const int32_t* slen, uint8_t* tmp, size_t tmp_cap,
                           uint64_t* coff, int32_t* clen, size_t nb, int max_src_len, int hc_level)
{
    if (hc_level <= 0) {
        uint64_t total = 0;
        return b200lz4_compress_fast_compact_host(src, soff, slen, tmp, tmp_cap, coff, clen, nb, max_src_len, &total);
    }
    std::vector<int32_t> ccap(nb);
    uint64_t acc = 0;
    for (size_t i = 0; i < nb; i++) { coff[i] = acc; ccap[i] = (int32_t)b200::compress_bound((uint64_t)slen[i]); acc += b200::aligned_compress_bound((uint64_t)slen[i]); }
    if (acc > tmp_cap) return B200LZ4_E_ARG;
    return b200lz4_compress_hc_batch_host(src, soff, slen, tmp, coff, ccap.data(), clen, nb, hc_level);
}

// ---------------------------------------------------------------- LZ4 Frame writer (frame_encode.cu)
namespace b200 {

// Where the FramePlan arrays of a call with nb blocks, ni items and nf frames lie in one blob, the same on the host and the
// device.  f_off, f_end and the two carry words come last: one copy brings the results back.
struct FramePlanLayout {
    size_t b_soff, b_slen, b_slot, b_ccap, b_clen, b_poff, b_plen, b_sum;
    size_t i_frame, i_block, i_size, i_off;
    size_t f_soff, f_len, f_len32, f_sum, f_off, f_end, carry, bytes = 0;
    FramePlanLayout(size_t nb, size_t ni, size_t nf)
    {
        auto take = [&](size_t n) { const size_t at = bytes; bytes = (bytes + n + 15) & ~size_t(15); return at; };
        b_soff = take(8 * nb); b_slen = take(4 * nb); b_slot = take(8 * nb); b_ccap = take(4 * nb); b_clen = take(4 * nb);
        b_poff = take(8 * nb); b_plen = take(4 * nb); b_sum = take(4 * nb);
        i_frame = take(4 * ni); i_block = take(4 * ni); i_size = take(4 * ni); i_off = take(8 * ni);
        f_soff = take(8 * nf); f_len = take(8 * nf); f_len32 = take(4 * nf); f_sum = take(4 * nf);
        f_off = take(8 * nf); f_end = take(8 * nf); carry = take(16);
    }
};

struct FrameChunk { size_t i0, i1, b0, b1; };                       // items [i0, i1), their blocks [b0, b1)

static int64_t compress_frames_dev(const uint8_t* d_src, const uint64_t* src_off, const uint64_t* src_len, size_t nf,
                                   uint8_t* d_dst, size_t dst_capacity, uint64_t* frame_off, uint64_t* frame_len,
                                   int bsCode, int flags, int hc_level, cudaStream_t st)
{
    // ---- arguments and sizes: nothing is launched or written before these pass
    if (bsCode < 4 || bsCode > 7) return fail_arg("bsCode must be 4..7");
    if (nf == 0) return 0;
    if (!src_off || !src_len || !d_dst) return fail_arg("null pointer");
    const uint64_t bs = 1ull << (8 + 2 * bsCode);
    uint64_t need = 0, nb = 0, ni = 0, bytes = 0;
    bool too_long = false;
    for (size_t f = 0; f < nf; f++) {
        const uint64_t n = src_len[f];
        if (n > (1ull << 47)) return fail_arg("src_len");
        need += b200lz4f_compress_bound(n, bsCode);
        nb += (n + bs - 1) / bs; ni += n ? (n + bs - 1) / bs : 1; bytes += n;
        if ((flags & 1) && n > 0x7FFFFFFFull) too_long = true;
    }
    if (bytes && !d_src) return fail_arg("null pointer");
    if (ni > 0x7FFFFFFFull) return fail_arg("too many blocks in one call");
    if (need > dst_capacity) return -9;
    if (too_long) return -10;                                       // the content checksum kernel takes 31-bit lengths (f_len32)
    FrameScratch* s; SideStream* side; int rc = get_frame_scratch(&s, &side); if (rc) return rc;
    const FramePlanLayout L(nb, ni, nf);
    rc = reserve_pinned(s->h_plan, s->h_plan_cap, L.bytes);
    if (!rc) rc = reserve_device(s->d_plan, s->plan_cap, L.bytes);
    if (rc) return rc;

    // ---- plan: blocks of bs bytes (the last one of a frame short), items, and chunks of at most CHUNK_SPAN source bytes and
    // CHUNK_BLOCKS items, so the compressed slots take the same room however large the call
    uint8_t* H = s->h_plan;
    auto h64 = [&](size_t o) { return (uint64_t*)(H + o); };
    auto h32 = [&](size_t o) { return (int32_t*)(H + o); };
    std::vector<FrameChunk> chunks;
    size_t b = 0, i = 0, ci0 = 0, cb0 = 0;
    uint64_t slot = 0, span = 0, slots_need = 0;
    for (size_t f = 0; f < nf; f++) {
        const uint64_t n = src_len[f], nbf = (n + bs - 1) / bs;
        h64(L.f_soff)[f] = src_off[f]; h64(L.f_len)[f] = n; h32(L.f_len32)[f] = (int32_t)(n < 0x7FFFFFFFull ? n : 0x7FFFFFFFull);
        for (uint64_t k = 0; k < (nbf ? nbf : 1); k++, i++) {
            const uint64_t len = nbf ? (n - k * bs < bs ? n - k * bs : bs) : 0;
            if (i > ci0 && (i - ci0 >= CHUNK_BLOCKS || span + len > CHUNK_SPAN)) {
                chunks.push_back(FrameChunk{ ci0, i, cb0, b });
                slots_need = slot > slots_need ? slot : slots_need;
                ci0 = i; cb0 = b; slot = 0; span = 0;
            }
            h32(L.i_frame)[i] = (int32_t)f;
            h32(L.i_block)[i] = nbf ? (int32_t)b : -1;
            if (!nbf) continue;
            h64(L.b_soff)[b] = src_off[f] + k * bs; h32(L.b_slen)[b] = (int32_t)len;
            h64(L.b_slot)[b] = slot; h32(L.b_ccap)[b] = (int32_t)compress_bound(len);
            slot += aligned_compress_bound(len); span += len; b++;
        }
    }
    chunks.push_back(FrameChunk{ ci0, i, cb0, b });
    slots_need = slot > slots_need ? slot : slots_need;
    h64(L.carry)[0] = 0;
    rc = reserve_device(s->d_slots, s->slots_cap, (size_t)slots_need + 16); if (rc) return rc;

    uint8_t* D = s->d_plan;
    const FramePlan P{ d_src, d_dst, s->d_slots,
                       (const uint64_t*)(D + L.b_soff), (const int32_t*)(D + L.b_slen), (const uint64_t*)(D + L.b_slot), (const int32_t*)(D + L.b_clen),
                       (uint64_t*)(D + L.b_poff), (int32_t*)(D + L.b_plen), (const uint32_t*)(D + L.b_sum),
                       (const uint32_t*)(D + L.i_frame), (const int32_t*)(D + L.i_block), (int32_t*)(D + L.i_size), (uint64_t*)(D + L.i_off),
                       (const uint64_t*)(D + L.f_len), (const uint32_t*)(D + L.f_sum), (uint64_t*)(D + L.f_off), (uint64_t*)(D + L.f_end),
                       (uint32_t)ni, bsCode, flags };
    uint64_t* carry = (uint64_t*)(D + L.carry);

    // ---- launches, all ordered after what `st` already holds
    Drain drain{ st, side->st };
    auto counted = [](cudaError_t e) { g_launch_count.fetch_add(1, std::memory_order_relaxed); return e; };
    CK(cudaMemcpyAsync(D, H, L.bytes, cudaMemcpyHostToDevice, st));
    if (flags & 1) {                // content checksums: the sources only, so from the start, beside everything else
        CK(cudaEventRecord(side->fork, st));
        CK(cudaStreamWaitEvent(side->st, side->fork, 0));
        CK(counted(launch_xxh32_long(d_src, (const uint64_t*)(D + L.f_soff), (const int32_t*)(D + L.f_len32), 0,
                                     (uint32_t*)(D + L.f_sum), nf, side->st)));
        CK(cudaEventRecord(side->join, side->st));
    }
    for (size_t k = 0; k < chunks.size(); k++) {
        const FrameChunk& c = chunks[k];
        if (c.b1 > c.b0) {          // the stream's compressor argument: hc_level 0 = the fast compressor, 1..17 = HC
            const BatchArgs a{ d_src, P.b_soff + c.b0, P.b_slen + c.b0, s->d_slots, P.b_slot + c.b0,
                               (const int32_t*)(D + L.b_ccap) + c.b0, (int32_t*)P.b_clen + c.b0, c.b1 - c.b0 };
            CK(counted(hc_level > 0 ? launch_compress_hc(a, hc_level, st) : launch_compress_fast(a, bs <= 65536 ? 65536 : 0, st)));
        }
        const uint32_t i0 = (uint32_t)c.i0, n = (uint32_t)(c.i1 - c.i0);
        CK(counted(launch_frame_sizes(P, i0, n, st)));
        CK(counted(launch_scan(P.i_size + i0, P.i_off + i0, carry + ((k + 1) & 1), carry + (k & 1), n, st)));
        CK(counted(launch_frame_emit(P, i0, n, st)));
    }
    if ((flags & 2) && nb) {        // block checksums over the payloads as written; the source average bounds the payloads'
        CK(counted((bytes / nb >= XXH_LONG_AVG ? launch_xxh32_long : launch_xxh32)(
            d_dst, P.b_poff, P.b_plen, 0, (uint32_t*)P.b_sum, (size_t)nb, st)));
    }
    if (flags & 1) CK(cudaStreamWaitEvent(st, side->join, 0));
    CK(counted(launch_frame_seal(P, st)));
    CK(cudaMemcpyAsync(H + L.f_off, D + L.f_off, L.bytes - L.f_off, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    drain.done = true;
    for (size_t f = 0; f < nf; f++) {
        if (frame_off) frame_off[f] = h64(L.f_off)[f];
        if (frame_len) frame_len[f] = h64(L.f_end)[f] - h64(L.f_off)[f];
    }
    return (int64_t)h64(L.carry)[chunks.size() & 1];
}

} // namespace b200

extern "C" {

size_t b200lz4f_compress_bound(size_t n, int bsCode)
{
    if (bsCode < 4 || bsCode > 7) return 0;
    const size_t bs = (size_t)1 << (8 + 2 * bsCode), nb = (n + bs - 1) / bs;
    return 4 + 2 + 8 + 1 + nb * 8 + n + 4 + 4;
}

int64_t b200lz4f_compress_dev(const uint8_t* d_src, const uint64_t* src_off, const uint64_t* src_len, size_t nf,
                              uint8_t* d_dst, size_t dst_capacity, uint64_t* frame_off, uint64_t* frame_len,
                              int bsCode, int flags, int hc_level, void* stream)
{
    return b200::compress_frames_dev(d_src, src_off, src_len, nf, d_dst, dst_capacity, frame_off, frame_len, bsCode, flags,
                                     hc_level, (cudaStream_t)stream);
}

// The device writer on a copy of src in the thread's staging buffer: the source at its own 16-byte phase (the fast
// compressor's chunks, and so its streams, follow the source's alignment), the frame behind it.
int64_t b200lz4f_compress_host_hc(const uint8_t* src, size_t n, uint8_t* dst, size_t cap, int bsCode, int flags, int hc_level)
{
    if (bsCode < 4 || bsCode > 7) return b200::fail_arg("bsCode must be 4..7");
    const size_t bound = b200lz4f_compress_bound(n, bsCode);
    if (cap < bound) return -9;
    b200::FrameScratch* s; cudaStream_t st;
    int rc = b200::get_frame_scratch(&s, nullptr, &st); if (rc) return rc;
    const uint64_t phase = (uintptr_t)src & 15, len = n, at = (phase + n + 15) & ~uint64_t(15);
    rc = b200::reserve_device(s->d_stage, s->stage_cap, at + bound); if (rc) return rc;
    b200::Drain drain{ st };
    CK(cudaMemcpyAsync(s->d_stage + phase, src, n, cudaMemcpyHostToDevice, st));
    const int64_t w = b200::compress_frames_dev(s->d_stage, &phase, &len, 1, s->d_stage + at, bound, nullptr, nullptr, bsCode,
                                                flags, hc_level, st);
    if (w < 0) return w;
    CK(cudaMemcpyAsync(dst, s->d_stage + at, (size_t)w, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    drain.done = true;
    return w;
}
int64_t b200lz4f_compress_host(const uint8_t* src, size_t n, uint8_t* dst, size_t cap, int bsCode, int flags)
{ return b200lz4f_compress_host_hc(src, n, dst, cap, bsCode, flags, 0); }

// ---------------------------------------------------------------- "LZ4Block" container
static const uint8_t LZ4BLOCK_MAGIC[8] = { 'L', 'Z', '4', 'B', 'l', 'o', 'c', 'k' };
enum { LZ4BLOCK_HEADER = 8 + 1 + 4 + 4 + 4, METHOD_RAW = 0x10, METHOD_LZ4 = 0x20 };
static const uint32_t LZ4BLOCK_SEED = 0x9747b28cu;                               // LZ4BlockOutputStream.java:56

static int lz4block_level(int blockSize)                                        // LZ4BlockOutputStream.java:58-70
{
    int lvl = 0; while ((1 << lvl) < blockSize) lvl++;                           // 32 - numberOfLeadingZeros(blockSize - 1)
    lvl -= 10; return lvl < 0 ? 0 : lvl;
}

size_t b200lz4block_compress_bound(size_t n, int blockSize)
{
    if (blockSize < 64 || blockSize > (1 << 25)) return 0;
    const size_t nb = (n + blockSize - 1) / blockSize;
    return (nb + 1) * LZ4BLOCK_HEADER + n + nb * 16 + n / 255;
}

int64_t b200lz4block_compress_host_hc(const uint8_t* src, size_t n, uint8_t* dst, size_t cap, int blockSize, int hc_level)
{
    if (blockSize < 64 || blockSize > (1 << 25)) return B200LZ4_E_ARG;
    if (cap < b200lz4block_compress_bound(n, blockSize)) return -9;
    const int level = lz4block_level(blockSize);
    const size_t bs = (size_t)blockSize, nb = (n + bs - 1) / bs;
    size_t o = 0;
    if (nb) {
        std::vector<uint64_t> soff(nb), coff(nb);
        std::vector<int32_t> slen(nb), clen(nb);
        std::vector<uint32_t> sums(nb);
        for (size_t i = 0; i < nb; i++) { soff[i] = i * bs; slen[i] = (int32_t)((n - i * bs) < bs ? (n - i * bs) : bs); }
        size_t tmp_cap = 0; for (size_t i = 0; i < nb; i++) tmp_cap += (size_t)slen[i] + slen[i] / 255 + 32;
        uint8_t* tmp = (uint8_t*)malloc(tmp_cap ? tmp_cap : 1);
        if (!tmp) return B200LZ4_E_ARG;
        int rc = compress_blocks(src, soff.data(), slen.data(), tmp, tmp_cap, coff.data(), clen.data(), nb, bs <= 65536 ? 65536 : 0, hc_level);
        if (!rc) rc = b200xxh32_batch_host(src, soff.data(), slen.data(), LZ4BLOCK_SEED, sums.data(), nb);   // checksum of the ORIGINAL bytes
        if (rc) { free(tmp); return rc; }
        for (size_t i = 0; i < nb; i++) {                                        // flushBufferedData (:203-227)
            const bool raw = clen[i] <= 0 || clen[i] >= slen[i];
            const uint32_t sz = raw ? (uint32_t)slen[i] : (uint32_t)clen[i];
            memcpy(dst + o, LZ4BLOCK_MAGIC, 8);
            dst[o + 8] = (uint8_t)((raw ? METHOD_RAW : METHOD_LZ4) | level);
            put32(dst + o + 9, sz); put32(dst + o + 13, (uint32_t)slen[i]);
            put32(dst + o + 17, sums[i] & 0x0FFFFFFFu);                          // Checksum view keeps 28 bits (StreamingXXHash32.java:106)
            memcpy(dst + o + LZ4BLOCK_HEADER, raw ? src + soff[i] : tmp + coff[i], sz);
            o += LZ4BLOCK_HEADER + sz;
        }
        free(tmp);
    }
    memcpy(dst + o, LZ4BLOCK_MAGIC, 8);                                          // finish(): empty block (:255-266)
    dst[o + 8] = (uint8_t)(METHOD_RAW | level);
    put32(dst + o + 9, 0); put32(dst + o + 13, 0); put32(dst + o + 17, 0);
    o += LZ4BLOCK_HEADER;
    return (int64_t)o;
}
int64_t b200lz4block_compress_host(const uint8_t* src, size_t n, uint8_t* dst, size_t cap, int blockSize)
{ return b200lz4block_compress_host_hc(src, n, dst, cap, blockSize, 0); }

// Decodes an LZ4Block stream the way LZ4BlockInputStream reads it.  stopOnEmptyBlock != 0 (the reference's default, :100-104):
// reading ends at the first empty block, whatever follows is left alone (*srcConsumed says where), and a stream that ends
// before one is "Stream ended prematurely" (:192-198).  stopOnEmptyBlock == 0: empty blocks are stepped over, concatenated
// streams continue, and the end of src at (or inside) a header ends the stream quietly (:193-194, tryReadFully).
// Returns decoded bytes; -1 premature end, -2 "Stream is corrupted", -9 dst too small.
int64_t b200lz4block_decompress_host(const uint8_t* src, size_t n, uint8_t* dst, size_t cap, int stopOnEmptyBlock, size_t* srcConsumed)
{
    std::vector<uint64_t> soff, doff; std::vector<int32_t> savail, dlen, csz; std::vector<uint32_t> want;
    std::vector<uint64_t> hoff; std::vector<int32_t> hlen;
    size_t ip = 0, op = 0;
    int64_t tail = 0;                    // what is wrong with the container itself, behind the blocks collected so far: the reader
                                         // would have decoded and checked THOSE first, so their verdict comes first
    for (;;) {                                                                   // refill (:191-264)
        if (n - ip < LZ4BLOCK_HEADER) { if (stopOnEmptyBlock) tail = -1; else ip = n; break; }
        if (memcmp(src + ip, LZ4BLOCK_MAGIC, 8) != 0) { tail = -2; break; }
        const int token = src[ip + 8], method = token & 0xF0, level = 10 + (token & 0x0F);
        if (method != METHOD_RAW && method != METHOD_LZ4) { tail = -2; break; }
        const int32_t clen = (int32_t)get32(src + ip + 9), olen = (int32_t)get32(src + ip + 13);
        const uint32_t check = get32(src + ip + 17);
        if (olen > (1 << level) || olen < 0 || clen < 0 || (olen == 0 && clen != 0) || (olen != 0 && clen == 0) ||
            (method == METHOD_RAW && olen != clen)) { tail = -2; break; }
        ip += LZ4BLOCK_HEADER;
        if (olen == 0) { if (check != 0) { tail = -2; break; } if (stopOnEmptyBlock) break; continue; }   // empty block (:225-233)
        if (n - ip < (size_t)clen) { tail = -1; break; }
        if (cap - op < (size_t)olen) { tail = -9; break; }
        if (method == METHOD_RAW) memcpy(dst + op, src + ip, (size_t)olen);
        else { soff.push_back(ip); savail.push_back(clen); doff.push_back(op); dlen.push_back(olen); csz.push_back(clen); }
        hoff.push_back(op); hlen.push_back(olen); want.push_back(check);
        ip += (size_t)clen; op += (size_t)olen;
    }
    // per block the reader decodes, compares the consumed length, then the checksum -- all "Stream is corrupted" (:236-262)
    if (!soff.empty()) {
        std::vector<int32_t> res(soff.size());
        int rc = b200lz4_decompress_fast_batch_host(src, soff.data(), savail.data(), dst, doff.data(), dlen.data(), res.data(), soff.size());
        if (rc) return rc;
        for (size_t i = 0; i < res.size(); i++) if (res[i] != csz[i]) return -2;  // compressedLen != compressedLen2 (:247-250)
    }
    if (!hoff.empty()) {
        std::vector<uint32_t> sums(hoff.size());
        int rc = b200xxh32_batch_host(dst, hoff.data(), hlen.data(), LZ4BLOCK_SEED, sums.data(), hoff.size());
        if (rc) return rc;
        for (size_t i = 0; i < sums.size(); i++) if ((sums[i] & 0x0FFFFFFFu) != want[i]) return -2;
    }
    if (tail) return tail;
    if (srcConsumed) *srcConsumed = ip;
    return (int64_t)op;
}

// ---------------------------------------------------------------- length-prefixed block (LZ4CompressorWithLength.java:45-50)
int b200lz4_compress_with_length(const char* src, char* dst, int srcSize, int dstCapacity)
{
    if (dstCapacity < 4) return 0;
    const int r = b200lz4_compress_default(src, dst + 4, srcSize, dstCapacity - 4);
    if (r <= 0) return r;
    put32((uint8_t*)dst, (uint32_t)srcSize);
    return r + 4;
}
int b200lz4_decompressed_length(const char* src) { return (int)get32((const uint8_t*)src); }   // LZ4DecompressorWithLength.java:52-54
// fast-decompressor flavour: returns bytes read (incl. the 4-byte prefix) or < 0 (LZ4DecompressorWithLength.java:125-131)
int b200lz4_decompress_with_length(const char* src, int srcAvail, char* dst, int dstCapacity)
{
    if (srcAvail < 4) return -1;
    const int n = b200lz4_decompressed_length(src);
    if (n < 0 || n > dstCapacity) return -1;
    const int r = b200lz4_decompress_fast_bounded(src + 4, srcAvail - 4, dst, n);
    return r < 0 ? r : r + 4;
}

} // extern "C"
