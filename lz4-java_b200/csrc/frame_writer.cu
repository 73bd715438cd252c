// frame_writer.cu — the device half of the incremental frame writer (b200lz4f_writer_write_dev: frame_writer_write_dev in
// containers.cu).  Each of ns streams is one LZ4FrameOutputStream whose content arrives in pieces; the host plans a call from
// the lengths, ops, room and carried states alone (which whole blocks, which short block at a flush, whether the header or
// the EndMark is due), and the call runs the frame writer's chunk loop (compress_frames_dev, frame_encode.cu) with these
// item kernels in place of frame_encode.cu's:
//   frame_writer_size_kernel   the bytes every item takes: block word, stored or compressed payload, block checksum slot; the
//                              header on a stream's first item of its first call, EndMark and content checksum on its last
//                              item of the closing call
//   frame_writer_emit_kernel   block words and payloads, one warp per block, each stream's items from the start of its range
// and once per call, behind the block checksums and the carried content checksums (launch_xxh32_long_carry, on a second
// stream from the start):
//   frame_writer_seal_kernel   headers with the declared content size, block checksums, EndMarks, content checksum digests,
//                              and each stream's range written
#include "common.cuh"
#include "kernels.h"
#include "frame_header.cuh"

namespace b200 {

__device__ __forceinline__ bool writer_head(const FrameWriterPlan& w, uint32_t i)
{
    return (w.f_mode[w.p.i_frame[i]] & WRITER_HEAD) && item_first(w.p, i);
}

// one thread per item of [i0, i0 + n)
__global__ void __launch_bounds__(256)
frame_writer_size_kernel(const FrameWriterPlan w, uint32_t i0, uint32_t n)
{
    const uint32_t t = blockIdx.x * 256 + threadIdx.x;
    if (t >= n) return;
    const FramePlan& p = w.p;
    const uint32_t i = i0 + t;
    const int32_t b = p.i_block[i];
    int32_t size = 0;
    if (b >= 0) {
        const int32_t slen = p.b_slen[b], clen = p.b_clen[b];
        size = 4 + (block_stored(clen, slen) ? slen : clen) + ((p.flags & 2) ? 4 : 0);
    }
    if (writer_head(w, i)) size += frame_header_bytes(p.flags);
    if (writer_tail(w, i)) size += frame_tail_bytes(p.flags);
    p.i_size[i] = size;
}

// one warp per item of [i0, i0 + n): its block word and payload (the compressed slot, or the source when stored)
__global__ void __launch_bounds__(128)
frame_writer_emit_kernel(const FrameWriterPlan w, uint32_t i0, uint32_t n)
{
    const uint32_t t = blockIdx.x * 4 + (threadIdx.x >> 5);
    if (t >= n) return;
    const FramePlan& p = w.p;
    const uint32_t i = i0 + t;
    const int32_t b = p.i_block[i];
    if (b < 0) return;                                                  // the header or the EndMark alone
    const int lane = lane_id();
    const int32_t slen = p.b_slen[b], clen = p.b_clen[b];
    const bool stored = block_stored(clen, slen);
    const int32_t sz = stored ? slen : clen;
    const uint64_t pos = writer_item_pos(w, i) + (writer_head(w, i) ? frame_header_bytes(p.flags) : 0);
    uint8_t* d = p.dst + pos;
    const uint32_t word = (uint32_t)sz | (stored ? 0x80000000u : 0u);
    if (lane < 4) d[lane] = (uint8_t)(word >> (8 * lane));
    warp_copy(d + 4, stored ? p.src + p.b_soff[b] : p.slots + p.b_slot[b], sz, lane);
    if (lane == 0 && (p.flags & 2)) { p.b_poff[b] = pos + 4; p.b_plen[b] = sz; }
}

// one thread per item of the call, after every chunk and checksum
__global__ void __launch_bounds__(256)
frame_writer_seal_kernel(const FrameWriterPlan w)
{
    const FramePlan& p = w.p;
    const uint32_t i = blockIdx.x * 256 + threadIdx.x;
    if (i >= p.nitems) return;
    const uint32_t f = p.i_frame[i];
    const int32_t b = p.i_block[i];
    if (b >= 0 && (p.flags & 2)) put_le32(p.dst + p.b_poff[b] + (uint32_t)p.b_plen[b], p.b_sum[b]);
    const uint64_t start = writer_item_pos(w, i), end = start + (uint64_t)p.i_size[i];
    if (writer_head(w, i)) frame_write_header(p.dst + start, p.bsCode, p.flags, p.f_len[f]);   // writeHeader (:178-190)
    if (writer_tail(w, i)) {                                            // writeEndMark (:243-249)
        uint8_t* e = p.dst + end - frame_tail_bytes(p.flags);
        put_le32(e, 0);
        if (p.flags & 1) put_le32(e + 4, p.f_sum[f]);
    }
    if (item_last(p, i)) { p.f_off[f] = w.f_doff[f]; p.f_end[f] = end; }
}

// launchers: the same code in the emulator build (B200_LAUNCH)
cudaError_t launch_frame_writer_sizes(const FrameWriterPlan& w, uint32_t i0, uint32_t n, cudaStream_t st)
{
    if (n == 0) return cudaSuccess;
    B200_LAUNCH(frame_writer_size_kernel, (n + 255) / 256, 256, st, w, i0, n);
    return cudaGetLastError();
}
cudaError_t launch_frame_writer_emit(const FrameWriterPlan& w, uint32_t i0, uint32_t n, cudaStream_t st)
{
    if (n == 0) return cudaSuccess;
    B200_LAUNCH(frame_writer_emit_kernel, (n + 3) / 4, 128, st, w, i0, n);
    return cudaGetLastError();
}
cudaError_t launch_frame_writer_seal(const FrameWriterPlan& w, cudaStream_t st)
{
    if (w.p.nitems == 0) return cudaSuccess;
    B200_LAUNCH(frame_writer_seal_kernel, (w.p.nitems + 255) / 256, 256, st, w);
    return cudaGetLastError();
}

} // namespace b200
