// frame_encode.cu — the device half of the LZ4 Frame writer (compress_frames_dev in containers.cu, behind
// b200lz4f_compress_dev and b200lz4f_compress_host_hc): what LZ4FrameOutputStream.writeHeader / writeBlock / writeEndMark
// write (LZ4FrameOutputStream.java:178-251), for many frames whose bytes are in device memory.  The host only plans (blocks,
// items, chunks: no payload byte is touched).  The blocks are compressed by the library's batch compressors into bound-sized
// slots one chunk at a time, and per chunk
//   frame_size_kernel    the bytes every item takes in its frame (block word, stored or compressed payload, block
//                        checksum slot; the header on a frame's first item, EndMark and content checksum on its last)
//   compact_scan_kernel  where every item goes (compact.cu), the running offset carried from chunk to chunk on the device
//   frame_emit_kernel    block words and payloads, one warp per block
// and once per call, behind the block checksums (launch_xxh32*, over the payloads as written) and the content checksums
// (launch_xxh32_long over each frame's source, on a second stream from the start):
//   frame_seal_kernel    magic, descriptor, header checksum byte, block checksums, EndMark, content checksum
#include "common.cuh"
#include "kernels.h"
#include "frame_header.cuh"

namespace b200 {

// one thread per item of [i0, i0 + n)
__global__ void __launch_bounds__(256)
frame_size_kernel(const FramePlan p, uint32_t i0, uint32_t n)
{
    const uint32_t t = blockIdx.x * 256 + threadIdx.x;
    if (t >= n) return;
    const uint32_t i = i0 + t;
    const int32_t b = p.i_block[i];
    int32_t size = 0;
    if (b >= 0) {
        const int32_t slen = p.b_slen[b], clen = p.b_clen[b];
        size = 4 + (block_stored(clen, slen) ? slen : clen) + ((p.flags & 2) ? 4 : 0);
    }
    if (item_first(p, i)) size += frame_header_bytes(p.flags);
    if (item_last(p, i)) size += frame_tail_bytes(p.flags);
    p.i_size[i] = size;
}

// one warp per item of [i0, i0 + n): its block word and payload (the compressed slot, or the source when stored)
__global__ void __launch_bounds__(128)
frame_emit_kernel(const FramePlan p, uint32_t i0, uint32_t n)
{
    const uint32_t t = blockIdx.x * 4 + (threadIdx.x >> 5);
    if (t >= n) return;
    const uint32_t i = i0 + t;
    const int32_t b = p.i_block[i];
    if (b < 0) return;                                                  // an empty frame: header and EndMark only
    const int lane = lane_id();
    const int32_t slen = p.b_slen[b], clen = p.b_clen[b];
    const bool stored = block_stored(clen, slen);
    const int32_t sz = stored ? slen : clen;
    const uint64_t pos = p.i_off[i] + (item_first(p, i) ? frame_header_bytes(p.flags) : 0);
    uint8_t* d = p.dst + pos;
    const uint32_t word = (uint32_t)sz | (stored ? 0x80000000u : 0u);
    if (lane < 4) d[lane] = (uint8_t)(word >> (8 * lane));
    warp_copy(d + 4, stored ? p.src + p.b_soff[b] : p.slots + p.b_slot[b], sz, lane);
    if (lane == 0 && (p.flags & 2)) { p.b_poff[b] = pos + 4; p.b_plen[b] = sz; }
}

// one thread per item of the call, after every chunk and checksum
__global__ void __launch_bounds__(256)
frame_seal_kernel(const FramePlan p)
{
    const uint32_t i = blockIdx.x * 256 + threadIdx.x;
    if (i >= p.nitems) return;
    const uint32_t f = p.i_frame[i];
    const int32_t b = p.i_block[i];
    if (b >= 0 && (p.flags & 2)) put_le32(p.dst + p.b_poff[b] + (uint32_t)p.b_plen[b], p.b_sum[b]);
    const uint64_t start = p.i_off[i], end = start + (uint64_t)p.i_size[i];
    if (item_first(p, i)) {                                             // writeHeader (:178-190)
        uint8_t* h = p.dst + start;
        put_le32(h, 0x184D2204u);
        const int dl = frame_descriptor(h + 4, p.bsCode, p.flags, p.f_len[f]);
        h[4 + dl] = (uint8_t)(xxh32_short(h + 4, dl) >> 8);
        p.f_off[f] = start;
    }
    if (item_last(p, i)) {                                              // writeEndMark (:243-249)
        uint8_t* e = p.dst + end - frame_tail_bytes(p.flags);
        put_le32(e, 0);
        if (p.flags & 1) put_le32(e + 4, p.f_sum[f]);
        p.f_end[f] = end;
    }
}

// launchers: the same code in the emulator build (B200_LAUNCH)
cudaError_t launch_frame_sizes(const FramePlan& p, uint32_t i0, uint32_t n, cudaStream_t st)
{
    if (n == 0) return cudaSuccess;
    B200_LAUNCH(frame_size_kernel, (n + 255) / 256, 256, st, p, i0, n);
    return cudaGetLastError();
}
cudaError_t launch_frame_emit(const FramePlan& p, uint32_t i0, uint32_t n, cudaStream_t st)
{
    if (n == 0) return cudaSuccess;
    B200_LAUNCH(frame_emit_kernel, (n + 3) / 4, 128, st, p, i0, n);
    return cudaGetLastError();
}
cudaError_t launch_frame_seal(const FramePlan& p, cudaStream_t st)
{
    if (p.nitems == 0) return cudaSuccess;
    B200_LAUNCH(frame_seal_kernel, (p.nitems + 255) / 256, 256, st, p);
    return cudaGetLastError();
}

} // namespace b200
