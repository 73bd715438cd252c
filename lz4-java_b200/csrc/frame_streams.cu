// frame_streams.cu — the device half of b200lz4f_decompress_streams_dev (frame_streams_decompress_dev in frame.cu): many
// independent LZ4 frame streams in device memory, each read as its own LZ4FrameInputStream(in, readSingleFrame), with one
// result per stream.  Every per-block and per-frame fact stays on the device:
//   frame_streams_walk_kernel     one thread per stream runs the container walk (walk_frames, kernels.h, the indexers' walk
//                                 too): first counting frames, blocks, checksums and slot bytes, then, behind scans of the
//                                 counts, writing decode_dev's descriptor arrays for the whole call
//   (decode_dev's payload launches: XXH32 of descriptors and checksummed blocks, the gather of stored blocks and the safe
//    decoder into the slots, the chained content checksums beside it)
//   frame_streams_verdict_kernel  one warp per stream: decode_dev's stream-order checks frame by frame, the tail code and the
//                                 room, then where each block of a stream that passed goes in d_dst
// and one gather packs the verified blocks.  A stream is walked by one thread, twice: one long stream of many small blocks is a
// serial chain of dependent loads (b200lz4f_decompress_dev with hints is the call for one large container).
#include "common.cuh"
#include "kernels.h"

namespace b200 {

// The counting walk's sink: per stream the FS_* counts (kernels.h), slots in 16-byte units (every slot is a multiple of 16).
struct FrameStreamCountSink {
    uint64_t n[FS_ROWS] = {}; uint32_t bs = 0; uint8_t flg = 0;
    __device__ void frame_begin(const WalkFrame& w) { flg = w.flg; bs = 1u << (8 + 2 * (w.bd >> 4)); }
    __device__ void block(uint64_t, uint32_t word, uint32_t)
    {
        const uint32_t size = word & 0x7FFFFFFFu; const bool raw = word >> 31;
        n[raw ? FS_RAW : FS_COMP]++;
        if (flg & 0x10) n[FS_BSUM]++;
        n[FS_SLOT16] += frame_slot_bytes(frame_slot_room(bs, size, raw), bs) >> 4;
    }
    __device__ void frame_end(const WalkFrame& w) { n[FS_FRAME]++; if (w.has_checksum) n[FS_FSUM]++; }
};

// The recording walk's sink: what build_descriptors (frame.cu) lays out for an index, for every stream of the call at once.
// c, q, b, k, f, j: the stream's next compressed, stored, any and checksummed block, its next frame and content-checksummed
// frame (exclusive prefixes of the counts); slot: the next slot byte.
struct FrameStreamRecordSink {
    const FrameStreamRead& r; uint64_t soff, c, q, b, k, f, j, slot;
    uint64_t first = 0; int32_t bsum0 = -1; uint32_t bs = 0; uint8_t flg = 0;
    __device__ void frame_begin(const WalkFrame& w)
    {
        flg = w.flg; bs = 1u << (8 + 2 * (w.bd >> 4));
        first = b; bsum0 = (flg & 0x10) ? (int32_t)k : -1;
    }
    __device__ void block(uint64_t at, uint32_t word, uint32_t checksum)
    {
        const uint32_t size = word & 0x7FFFFFFFu; const bool raw = word >> 31;
        const uint64_t room = frame_slot_room(bs, size, raw);
        r.k_off[b] = slot;
        if (raw) {
            r.k_comp[b] = -1; r.k_rawlen[b] = (int32_t)size;
            r.r_soff[q] = soff + at; r.r_doff[q] = slot; r.r_len[q++] = (int32_t)size;
        } else {
            r.k_comp[b] = (int32_t)c; r.k_rawlen[b] = 0;
            r.c_soff[c] = soff + at; r.c_doff[c] = slot; r.c_slen[c] = (int32_t)size; r.c_dcap[c++] = (int32_t)room;
        }
        if (flg & 0x10) { r.b_off[k] = soff + at; r.b_len[k] = (int32_t)size; r.b_want[k++] = checksum; }
        slot += frame_slot_bytes(room, bs);
        b++;
    }
    __device__ void frame_end(const WalkFrame& w)
    {
        r.h_off[f] = soff + w.desc_off; r.h_len[f] = w.desc_len;
        r.fr_first[f] = (uint32_t)first; r.fr_nblk[f] = (uint32_t)(b - first); r.fr_bsum[f] = bsum0;
        r.fr_size[f] = w.content_size; r.fr_bits[f] = (uint32_t)w.hc_byte | (w.has_size ? 0x100u : 0u);
        r.fr_fsum[f] = -1;
        if (w.has_checksum) {
            r.f_first[j] = (uint32_t)first; r.f_nblk[j] = (uint32_t)(b - first); r.f_want[j] = w.content_checksum;
            r.fr_fsum[f] = (int32_t)j++;
        }
        f++;
    }
};

__global__ void __launch_bounds__(128)
frame_streams_walk_kernel(const FrameStreamRead r, bool record)
{
    const uint32_t s = blockIdx.x * 128 + threadIdx.x;
    if (s >= r.ns) return;
    const uint8_t* src = r.src + r.s_off[s];
    const uint64_t n = r.s_len[s];
    if (!record) {
        FrameStreamCountSink sink;
        const WalkEnd e = walk_frames(src, n, 0, n, r.single, sink);
        bool over = false;
        for (int row = 0; row < FS_ROWS; row++) {
            const uint64_t v = sink.n[row];
            over |= v > 0x7FFFFFFFull;
            r.cnt[(size_t)row * r.ns + s] = (int32_t)(v > 0x7FFFFFFFull ? 0x7FFFFFFFull : v);
        }
        if (over) *r.over = 1;
        // index_verdict (frame.cu): an error before the first frame is the stream's result alone (there is nothing to
        // decode), one behind a frame is reported after what precedes it; no frame at all, skippable ones included, is -1
        r.tail[s] = e.err ? e.err : e.seen ? 0 : -1;
        r.ip[s] = e.ip;
        return;
    }
    auto at = [&](int row) { return r.pos[(size_t)row * r.ns + s]; };
    FrameStreamRecordSink sink{ r, r.s_off[s], at(FS_COMP), at(FS_RAW), at(FS_COMP) + at(FS_RAW), at(FS_BSUM), at(FS_FRAME),
                                at(FS_FSUM), at(FS_SLOT16) << 4 };
    walk_frames(src, n, 0, n, r.single, sink);
}

// decode_dev's verdict (frame.cu, the loop behind its synchronisation) for one stream per warp, 32 blocks at a time: frame by
// frame the descriptor hash (-3), block by block its checksum (-5) and its decode (-6), at the EndMark the content checksum
// (-7) and size (-8); then the walk's tail code, then the room (-9).  Then each block's place in d_dst: the stream's dst_off
// plus the decoded lengths before it, or length 0 for every block of a stream that failed.
__global__ void __launch_bounds__(128)
frame_streams_verdict_kernel(const FrameStreamRead r)
{
    const uint32_t s = blockIdx.x * 4 + (threadIdx.x >> 5);
    if (s >= r.ns) return;
    const int lane = lane_id();
    const size_t ns = r.ns;
    const uint64_t f0 = r.pos[FS_FRAME * ns + s], f1 = f0 + (uint64_t)r.cnt[FS_FRAME * ns + s];
    int32_t code = 0;
    uint64_t total = 0;
    for (uint64_t f = f0; f < f1 && !code; f++) {
        const uint32_t bits = r.fr_bits[f];
        if (((r.h_out[f] >> 8) & 0xFF) != (bits & 0xFF)) { code = -3; break; }
        const uint32_t first = r.fr_first[f], nblk = r.fr_nblk[f];
        const int32_t bsum0 = r.fr_bsum[f];
        uint64_t len = 0;
        for (uint32_t base = 0; base < nblk; base += 32) {
            const uint32_t k = base + (uint32_t)lane;
            int32_t bad = 0, l = 0;
            if (k < nblk) {
                const uint32_t b = first + k;
                if (bsum0 >= 0 && r.b_out[bsum0 + k] != r.b_want[bsum0 + k]) bad = -5;
                else {
                    const int32_t c = r.k_comp[b];
                    l = c < 0 ? r.k_rawlen[b] : r.c_res[c];
                    if (l < 0) { bad = -6; l = 0; }
                }
            }
            const uint32_t m = __ballot_sync(B200_FULL, bad != 0);
            if (m) { code = __shfl_sync(B200_FULL, bad, __ffs((int)m) - 1); break; }
            for (int d = 16; d; d >>= 1) l += __shfl_xor_sync(B200_FULL, l, d);
            len += (uint64_t)l;
        }
        if (code) break;
        const int32_t fs = r.fr_fsum[f];
        if (fs >= 0 && r.f_out[fs] != r.f_want[fs]) code = -7;
        else if ((bits & 0x100) && r.fr_size[f] != len) code = -8;
        total += len;
    }
    if (!code) code = r.tail[s];
    if (!code && total > r.d_cap[s]) code = -9;
    if (lane == 0) {
        r.result[s] = code ? (int64_t)code : (int64_t)total;
        r.consumed[s] = code ? 0 : r.ip[s];
        r.content[s] = (!code || code == -9) ? total : 0;
    }
    const uint64_t b0 = r.pos[FS_COMP * ns + s] + r.pos[FS_RAW * ns + s];
    const uint64_t b1 = b0 + (uint64_t)r.cnt[FS_COMP * ns + s] + (uint64_t)r.cnt[FS_RAW * ns + s];
    uint64_t run = r.d_off[s];
    for (uint64_t base = b0; base < b1; base += 32) {
        const uint64_t b = base + (uint64_t)lane;
        int32_t l = 0;
        if (b < b1 && !code) { const int32_t c = r.k_comp[b]; l = c < 0 ? r.k_rawlen[b] : r.c_res[c]; }
        int32_t x = l;                                                      // inclusive prefix over the lanes
        for (int d = 1; d < 32; d <<= 1) { const int32_t y = __shfl_up_sync(B200_FULL, x, d); if (lane >= d) x += y; }
        if (b < b1) { r.k_dst[b] = run + (uint64_t)(x - l); r.k_len[b] = l; }
        run += (uint64_t)__shfl_sync(B200_FULL, x, 31);
    }
}

// launchers: the same code in the emulator build (B200_LAUNCH)
cudaError_t launch_frame_streams_walk(const FrameStreamRead& r, bool record, cudaStream_t st)
{
    if (r.ns == 0) return cudaSuccess;
    B200_LAUNCH(frame_streams_walk_kernel, (r.ns + 127) / 128, 128, st, r, record);
    return cudaGetLastError();
}
cudaError_t launch_frame_streams_verdict(const FrameStreamRead& r, cudaStream_t st)
{
    if (r.ns == 0) return cudaSuccess;
    B200_LAUNCH(frame_streams_verdict_kernel, (r.ns + 3) / 4, 128, st, r);
    return cudaGetLastError();
}

} // namespace b200
