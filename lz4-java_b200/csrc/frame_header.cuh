// frame_header.cuh — what the two frame writers (frame_encode.cu, frame_writer.cu) write around the blocks: the header
// (LZ4FrameOutputStream.writeHeader, LZ4FrameOutputStream.java:178-191), the block word's stored bit and the EndMark
// (writeEndMark, :243-249); and the item placement both incremental writers (frame_writer.cu, lz4block.cu) share.
#pragma once
#include "common.cuh"
#include "kernels.h"

namespace b200 {

__device__ __forceinline__ int frame_header_bytes(int flags) { return 4 + 2 + ((flags & 4) ? 8 : 0) + 1; }   // magic FLG BD [size] HC
__device__ __forceinline__ int frame_tail_bytes(int flags) { return 4 + ((flags & 1) ? 4 : 0); }            // EndMark [checksum]
__device__ __forceinline__ bool item_first(const FramePlan& p, uint32_t i) { return i == 0 || p.i_frame[i - 1] != p.i_frame[i]; }
__device__ __forceinline__ bool item_last(const FramePlan& p, uint32_t i) { return i + 1 == p.nitems || p.i_frame[i + 1] != p.i_frame[i]; }
// stored as is when compression does not shrink the block (LZ4FrameOutputStream.java:215-222)
__device__ __forceinline__ bool block_stored(int32_t clen, int32_t slen) { return clen <= 0 || clen >= slen; }

// The incremental writers (frame_writer.cu, lz4block.cu): where item i lands, its stream's range then the bytes of the
// stream's items before it in this call; whether it carries the stream's end (the EndMark, or the LZ4Block end block)
__device__ __forceinline__ uint64_t writer_item_pos(const FrameWriterPlan& w, uint32_t i)
{
    const uint32_t f = w.p.i_frame[i];
    return w.f_doff[f] + (w.p.i_off[i] - w.p.i_off[w.f_first[f]]);
}
__device__ __forceinline__ bool writer_tail(const FrameWriterPlan& w, uint32_t i)
{
    return (w.f_mode[w.p.i_frame[i]] & WRITER_TAIL) && item_last(w.p, i);
}

__device__ __forceinline__ void put_le32(uint8_t* p, uint32_t v)
{
    p[0] = (uint8_t)v; p[1] = (uint8_t)(v >> 8); p[2] = (uint8_t)(v >> 16); p[3] = (uint8_t)(v >> 24);
}

// The frame descriptor writeHeader puts between the magic and the header checksum byte (LZ4FrameOutputStream.java:178-187):
// FLG, BD and, with flags bit 2, the 8-byte content size.  Returns the bytes written, 2 or 10.
__device__ __forceinline__ int frame_descriptor(uint8_t* d, int bsCode, int flags, uint64_t content_size)
{
    d[0] = (uint8_t)((1 << 6) | (1 << 5) | ((flags & 2) ? 1 << 4 : 0) | ((flags & 4) ? 1 << 3 : 0) | ((flags & 1) ? 1 << 2 : 0));
    d[1] = (uint8_t)(bsCode << 4);
    if (!(flags & 4)) return 2;
    for (int k = 0; k < 8; k++) d[2 + k] = (uint8_t)(content_size >> (8 * k));
    return 10;
}

// XXH32 with seed 0 of fewer than 16 bytes (the frame descriptor): no stripes, the tail and the avalanche of xxhash.c:290-348
__device__ __forceinline__ uint32_t xxh32_short(const uint8_t* p, int len)
{
    constexpr uint32_t P1 = 2654435761u, P2 = 2246822519u, P3 = 3266489917u, P4 = 668265263u, P5 = 374761393u;
    uint32_t h = P5 + (uint32_t)len;
    for (; len >= 4; p += 4, len -= 4) {
        const uint32_t w = p[0] | (p[1] << 8) | (p[2] << 16) | ((uint32_t)p[3] << 24);
        h = __funnelshift_l(h + w * P3, h + w * P3, 17) * P4;
    }
    for (; len > 0; p++, len--) h = __funnelshift_l(h + p[0] * P5, h + p[0] * P5, 11) * P1;
    h ^= h >> 15; h *= P2; h ^= h >> 13; h *= P3; h ^= h >> 16;
    return h;
}

// writeHeader at h (:178-191): magic, descriptor, header checksum byte
__device__ __forceinline__ void frame_write_header(uint8_t* h, int bsCode, int flags, uint64_t content_size)
{
    put_le32(h, 0x184D2204u);
    const int dl = frame_descriptor(h + 4, bsCode, flags, content_size);
    h[4 + dl] = (uint8_t)(xxh32_short(h + 4, dl) >> 8);
}

} // namespace b200
