// with_length.cu — the device halves of lz4-java's length-prefixed records (LZ4CompressorWithLength /
// LZ4DecompressorWithLength: 4 bytes of little-endian original length, then one LZ4 block) for many records whose bytes are
// in device memory (b200lz4_compress_with_length_dev / b200lz4_decompress_with_length_dev, driven from containers.cu).
// Writer: LZ4CompressorWithLength.compress (LZ4CompressorWithLength.java:45-50,155-158) on the frame writer's loop
// (compress_blocks_dev): its plan, chunks, compressed slots and carried scan, a record being one item and one block of its
// whole length, with per chunk
//   with_length_size_kernel  the bytes every record takes: 4 + the compressed block
//   with_length_emit_kernel  the length word and the block, one warp per record, and where the record lies
// Reader: LZ4DecompressorWithLength.decompress, either flavour (LZ4DecompressorWithLength.java:125-154), HBM to HBM:
//   with_length_head_kernel     one thread per record: the header checks of b200lz4_decompress_with_length{,_safe} and the
//                               decoder's arguments (a rejected record gets lengths that make the decoder touch nothing)
//   (the fast or the safe decoder over every record)
//   with_length_verdict_kernel  one thread per record: the header's -1, or the decoder's result (+4 for the fast flavour)
#include "common.cuh"
#include "kernels.h"

namespace b200 {

// one thread per item of [i0, i0 + n).  Bound-sized slots always hold the block, so clen > 0: there is no stored fallback.
__global__ void __launch_bounds__(256)
with_length_size_kernel(const FramePlan p, uint32_t i0, uint32_t n)
{
    const uint32_t t = blockIdx.x * 256 + threadIdx.x;
    if (t >= n) return;
    const uint32_t i = i0 + t;
    p.i_size[i] = 4 + p.b_clen[p.i_block[i]];
}

// one warp per item of [i0, i0 + n)
__global__ void __launch_bounds__(128)
with_length_emit_kernel(const FramePlan p, uint32_t i0, uint32_t n)
{
    const uint32_t t = blockIdx.x * 4 + (threadIdx.x >> 5);
    if (t >= n) return;
    const uint32_t i = i0 + t;
    const int32_t b = p.i_block[i];
    const int lane = lane_id();
    const int32_t clen = p.b_clen[b];
    const uint64_t at = p.i_off[i];
    uint8_t* d = p.dst + at;
    if (lane < 4) d[lane] = (uint8_t)((uint32_t)p.b_slen[b] >> (8 * lane));          // LZ4CompressorWithLength.java:155-158
    warp_copy(d + 4, p.slots + p.b_slot[b], clen, lane);
    if (lane == 0) { const uint32_t f = p.i_frame[i]; p.f_off[f] = at; p.f_end[f] = at + 4 + (uint64_t)clen; }
}

// ---- reader
__global__ void __launch_bounds__(128)
with_length_head_kernel(const WithLengthRead r)
{
    const uint32_t k = blockIdx.x * 128 + threadIdx.x;
    if (k >= r.n) return;
    const uint64_t at = r.s_off[k], len = r.s_len[k];
    int32_t declared = -1;
    bool ok = false;
    if (len >= 4) {                                                     // getDecompressedLength (LZ4DecompressorWithLength.java:52-54)
        declared = (int32_t)rd32(r.src + at);
        ok = declared >= 0 && (uint64_t)declared <= r.d_cap[k];
    }
    r.b_soff[k] = ok ? at + 4 : at;
    r.b_slen[k] = ok ? (int32_t)(len - 4) : 0;                          // fast: readable bytes; safe: the block's exact size
    r.b_dlen[k] = ok ? declared : 0;                                    // fast: the decoded size; safe: maxDestLen
    r.head[k] = ok ? 0 : -1;
    r.orig_len[k] = declared;
}

__global__ void __launch_bounds__(128)
with_length_verdict_kernel(const WithLengthRead r)
{
    const uint32_t k = blockIdx.x * 128 + threadIdx.x;
    if (k >= r.n) return;
    const int32_t res = r.b_res[k];
    r.result[k] = r.head[k] ? (int64_t)r.head[k] : (r.safe || res < 0) ? (int64_t)res : (int64_t)res + 4;
}

// launchers: the same code in the emulator build (B200_LAUNCH)
cudaError_t launch_with_length_sizes(const FramePlan& p, uint32_t i0, uint32_t n, cudaStream_t st)
{
    if (n == 0) return cudaSuccess;
    B200_LAUNCH(with_length_size_kernel, (n + 255) / 256, 256, st, p, i0, n);
    return cudaGetLastError();
}
cudaError_t launch_with_length_emit(const FramePlan& p, uint32_t i0, uint32_t n, cudaStream_t st)
{
    if (n == 0) return cudaSuccess;
    B200_LAUNCH(with_length_emit_kernel, (n + 3) / 4, 128, st, p, i0, n);
    return cudaGetLastError();
}
cudaError_t launch_with_length_head(const WithLengthRead& r, cudaStream_t st)
{
    if (r.n == 0) return cudaSuccess;
    B200_LAUNCH(with_length_head_kernel, (r.n + 127) / 128, 128, st, r);
    return cudaGetLastError();
}
cudaError_t launch_with_length_verdict(const WithLengthRead& r, cudaStream_t st)
{
    if (r.n == 0) return cudaSuccess;
    B200_LAUNCH(with_length_verdict_kernel, (r.n + 127) / 128, 128, st, r);
    return cudaGetLastError();
}

} // namespace b200
