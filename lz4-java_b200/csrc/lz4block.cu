// lz4block.cu — the device halves of lz4-java's "LZ4Block" stream writer and reader for many streams whose bytes are in
// device memory (b200lz4block_compress_dev / b200lz4block_decompress_dev, driven from containers.cu).
// Writer: LZ4BlockOutputStream.flushBufferedData / finish (LZ4BlockOutputStream.java:203-266) on the frame writer's loop
// (compress_blocks_dev): its plan, chunks, compressed slots and carried scan, with per chunk
//   lz4block_size_kernel    the bytes every item takes (header + stored or compressed payload; the end block on a stream's
//                           last item, alone for an empty stream)
//   lz4block_emit_kernel    magic, token, lengths and payload, one warp per block
// and once per call, behind the checksums of the ORIGINAL blocks (launch_xxh32*, seed 0x9747b28c, on the side stream from
// the start: they do not depend on the compressor)
//   lz4block_seal_kernel    the 28-bit checksums into the headers, the end blocks, where each stream lies
// Reader: LZ4BlockInputStream.refill (LZ4BlockInputStream.java:191-264), HBM to HBM.  Headers carry the original length, so
// every block's place in d_dst is known from the walk and blocks decode straight there:
//   lz4block_walk_kernel    one thread per stream walks its headers (walk_lz4block, kernels.h, the host reader's walk too):
//                           first counting, then, behind a scan of the counts, writing each block's record
//   (the fast decoder and the gather over the records, XXH32 of the decoded blocks)
//   lz4block_verdict_kernel one warp per stream: -2 if a block of it failed, else the walk's code or the decoded size
#include "common.cuh"
#include "kernels.h"

namespace b200 {

__device__ __forceinline__ bool lz4block_first(const FramePlan& p, uint32_t i) { return i == 0 || p.i_frame[i - 1] != p.i_frame[i]; }
__device__ __forceinline__ bool lz4block_last(const FramePlan& p, uint32_t i) { return i + 1 == p.nitems || p.i_frame[i + 1] != p.i_frame[i]; }
// stored as is when compression does not shrink the block (LZ4BlockOutputStream.java:210-218)
__device__ __forceinline__ bool lz4block_stored(int32_t clen, int32_t slen) { return clen <= 0 || clen >= slen; }

// magic, token (method | level), compressed and original length and checksum: 21 header bytes, one per lane
__device__ __forceinline__ uint8_t lz4block_header_byte(int k, int token, uint32_t clen, uint32_t olen, uint32_t check)
{
    if (k < 8) return (uint8_t)((k < 4 ? LZ4BLOCK_MAGIC_LO : LZ4BLOCK_MAGIC_HI) >> (8 * (k & 3)));
    if (k == 8) return (uint8_t)token;
    const uint32_t w = k < 13 ? clen : k < 17 ? olen : check;
    return (uint8_t)(w >> (8 * ((k - 9) & 3)));
}

// one thread per item of [i0, i0 + n)
__global__ void __launch_bounds__(256)
lz4block_size_kernel(const FramePlan p, uint32_t i0, uint32_t n)
{
    const uint32_t t = blockIdx.x * 256 + threadIdx.x;
    if (t >= n) return;
    const uint32_t i = i0 + t;
    const int32_t b = p.i_block[i];
    int32_t size = 0;
    if (b >= 0) {
        const int32_t slen = p.b_slen[b], clen = p.b_clen[b];
        size = LZ4BLOCK_HEADER + (lz4block_stored(clen, slen) ? slen : clen);
    }
    if (lz4block_last(p, i)) size += LZ4BLOCK_HEADER;
    p.i_size[i] = size;
}

// one warp per item of [i0, i0 + n): its header (the checksum left 0 for the seal) and payload
__global__ void __launch_bounds__(128)
lz4block_emit_kernel(const FramePlan p, uint32_t i0, uint32_t n)
{
    const uint32_t t = blockIdx.x * 4 + (threadIdx.x >> 5);
    if (t >= n) return;
    const uint32_t i = i0 + t;
    const int32_t b = p.i_block[i];
    if (b < 0) return;                                                  // an empty stream: its end block only
    const int lane = lane_id();
    const int32_t slen = p.b_slen[b], clen = p.b_clen[b];
    const bool stored = lz4block_stored(clen, slen);
    const int32_t sz = stored ? slen : clen;
    uint8_t* d = p.dst + p.i_off[i];
    if (lane < LZ4BLOCK_HEADER)
        d[lane] = lz4block_header_byte(lane, (stored ? LZ4BLOCK_RAW : LZ4BLOCK_LZ4) | p.level, (uint32_t)sz, (uint32_t)slen, 0);
    warp_copy(d + LZ4BLOCK_HEADER, stored ? p.src + p.b_soff[b] : p.slots + p.b_slot[b], sz, lane);
}

// one thread per item of the call, after every chunk and checksum
__global__ void __launch_bounds__(256)
lz4block_seal_kernel(const FramePlan p)
{
    const uint32_t i = blockIdx.x * 256 + threadIdx.x;
    if (i >= p.nitems) return;
    const uint32_t f = p.i_frame[i];
    const int32_t b = p.i_block[i];
    const uint64_t start = p.i_off[i], end = start + (uint64_t)p.i_size[i];
    if (b >= 0) {                                                       // the Checksum view keeps 28 bits (StreamingXXHash32.java:106)
        const uint32_t c = p.b_sum[b] & 0x0FFFFFFFu;
        uint8_t* h = p.dst + start + 17;
        h[0] = (uint8_t)c; h[1] = (uint8_t)(c >> 8); h[2] = (uint8_t)(c >> 16); h[3] = (uint8_t)(c >> 24);
    }
    if (lz4block_first(p, i)) p.f_off[f] = start;
    if (lz4block_last(p, i)) {                                          // finish(): the empty end block (:255-266)
        uint8_t* e = p.dst + end - LZ4BLOCK_HEADER;
        for (int k = 0; k < LZ4BLOCK_HEADER; k++) e[k] = lz4block_header_byte(k, LZ4BLOCK_RAW | p.level, 0, 0, 0);
        p.f_end[f] = end;
    }
}

// ---- reader
// The counting walk's sink: how many blocks of each method fit, and what the whole stream decodes to.
struct Lz4BlockCountSink {
    Lz4BlockRoom room; uint64_t content = 0; int32_t nc = 0, nr = 0;
    __device__ void block(uint64_t, bool raw, int32_t, int32_t olen, uint32_t)
    {
        content += (uint64_t)olen;
        if (room.take(olen)) (raw ? nr : nc)++;
    }
};

// The recording walk's sink: each block that fits, at its place in d_dst (the stream's dst_off + the lengths before it).
struct Lz4BlockRecordSink {
    const Lz4BlockRead& r; Lz4BlockRoom room; uint64_t soff, doff, c, q, k;     // next compressed, stored and any record
    __device__ void block(uint64_t at, bool raw, int32_t clen, int32_t olen, uint32_t check)
    {
        const uint64_t d = doff + room.used;
        if (!room.take(olen)) return;
        if (raw) { r.r_soff[q] = soff + at; r.r_doff[q] = d; r.r_len[q] = olen; q++; }
        else { r.c_soff[c] = soff + at; r.c_doff[c] = d; r.c_clen[c] = clen; r.c_olen[c] = olen; }
        r.b_doff[k] = d; r.b_len[k] = olen; r.b_want[k] = check; r.b_comp[k] = raw ? -1 : (int32_t)c;
        if (!raw) c++;
        k++;
    }
};

__global__ void __launch_bounds__(128)
lz4block_walk_kernel(const Lz4BlockRead r, bool record)
{
    const uint32_t s = blockIdx.x * 128 + threadIdx.x;
    if (s >= r.ns) return;
    const uint8_t* src = r.src + r.s_off[s];
    const uint64_t n = r.s_len[s];
    if (!record) {
        Lz4BlockCountSink sink{ Lz4BlockRoom{ r.d_cap[s] } };
        const Lz4BlockEnd e = walk_lz4block(src, n, r.stop, sink);
        r.n_comp[s] = sink.nc; r.n_raw[s] = sink.nr;
        r.tail[s] = sink.room.full ? -9 : e.err;                        // the block that does not fit comes before anything the walk met later
        r.ip[s] = e.ip; r.content[s] = sink.content;
        return;
    }
    Lz4BlockRecordSink sink{ r, Lz4BlockRoom{ r.d_cap[s] }, r.s_off[s], r.d_off[s], r.p_comp[s], r.p_raw[s], r.p_comp[s] + r.p_raw[s] };
    walk_lz4block(src, n, r.stop, sink);
}

// per block the reader decodes, compares the consumed length, then the checksum -- all "Stream is corrupted" (:236-262)
__global__ void __launch_bounds__(128)
lz4block_verdict_kernel(const Lz4BlockRead r)
{
    const uint32_t s = blockIdx.x * 4 + (threadIdx.x >> 5);
    if (s >= r.ns) return;
    const int lane = lane_id();
    const uint64_t k0 = r.p_comp[s] + r.p_raw[s], k1 = k0 + (uint64_t)r.n_comp[s] + (uint64_t)r.n_raw[s];
    bool bad = false;
    for (uint64_t base = k0; base < k1; base += 32) {
        const uint64_t k = base + (uint64_t)lane;
        bool b = false;
        if (k < k1) {
            const int32_t c = r.b_comp[k];
            b = (c >= 0 && r.c_res[c] != r.c_clen[c]) || (r.b_sum[k] & 0x0FFFFFFFu) != r.b_want[k];
        }
        if (__any_sync(B200_FULL, b)) { bad = true; break; }
    }
    if (lane == 0) {
        const int32_t tail = r.tail[s];
        const int64_t res = bad ? -2 : tail ? (int64_t)tail : (int64_t)r.content[s];
        r.result[s] = res;
        r.consumed[s] = res >= 0 ? r.ip[s] : 0;
    }
}

// launchers: the same code in the emulator build (B200_LAUNCH)
cudaError_t launch_lz4block_sizes(const FramePlan& p, uint32_t i0, uint32_t n, cudaStream_t st)
{
    if (n == 0) return cudaSuccess;
    B200_LAUNCH(lz4block_size_kernel, (n + 255) / 256, 256, st, p, i0, n);
    return cudaGetLastError();
}
cudaError_t launch_lz4block_emit(const FramePlan& p, uint32_t i0, uint32_t n, cudaStream_t st)
{
    if (n == 0) return cudaSuccess;
    B200_LAUNCH(lz4block_emit_kernel, (n + 3) / 4, 128, st, p, i0, n);
    return cudaGetLastError();
}
cudaError_t launch_lz4block_seal(const FramePlan& p, cudaStream_t st)
{
    if (p.nitems == 0) return cudaSuccess;
    B200_LAUNCH(lz4block_seal_kernel, (p.nitems + 255) / 256, 256, st, p);
    return cudaGetLastError();
}
cudaError_t launch_lz4block_walk(const Lz4BlockRead& r, bool record, cudaStream_t st)
{
    if (r.ns == 0) return cudaSuccess;
    B200_LAUNCH(lz4block_walk_kernel, (r.ns + 127) / 128, 128, st, r, record);
    return cudaGetLastError();
}
cudaError_t launch_lz4block_verdict(const Lz4BlockRead& r, cudaStream_t st)
{
    if (r.ns == 0) return cudaSuccess;
    B200_LAUNCH(lz4block_verdict_kernel, (r.ns + 3) / 4, 128, st, r);
    return cudaGetLastError();
}

} // namespace b200
