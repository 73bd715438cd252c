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
// Incremental writer (b200lz4block_writer_write_dev: lz4block_writer_write_dev in containers.cu): each stream is one
// LZ4BlockOutputStream whose content arrives in pieces.  The host plans a call as it plans the incremental frame writer's
// (writer_take), and the call runs the same chunk loop with
//   lz4block_writer_size_kernel  the bytes every item takes; the end block on a stream's last item of its closing call
//   lz4block_writer_emit_kernel  headers and payloads, one warp per block, each stream's items from the start of its range
//   lz4block_writer_seal_kernel  behind the checksums of the original blocks: checksums, end blocks, each stream's range
// Incremental reader (b200lz4block_reader_read_dev: lz4block_reader_read_dev in containers.cu): each stream is one
// LZ4BlockInputStream whose bytes arrive in pieces; a call takes the complete units at the start of each piece, and the only
// state carried between calls is the latched status:
//   lz4block_reader_walk_kernel     one thread per stream resumes the walk (walk_lz4block_from): first counting, then,
//                                   behind scans of the counts, writing each block's record, its place in d_dst exact
//   (the gather, the fast decoder and XXH32 of the decoded blocks, as for the whole-stream reader)
//   lz4block_reader_verdict_kernel  one warp per stream: cut at the first block that fails its decode or checksum
#include "common.cuh"
#include "kernels.h"
#include "frame_header.cuh"

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

// ---- incremental writer
// one thread per item of [i0, i0 + n)
__global__ void __launch_bounds__(256)
lz4block_writer_size_kernel(const FrameWriterPlan w, uint32_t i0, uint32_t n)
{
    const uint32_t t = blockIdx.x * 256 + threadIdx.x;
    if (t >= n) return;
    const FramePlan& p = w.p;
    const uint32_t i = i0 + t;
    const int32_t b = p.i_block[i];
    int32_t size = 0;
    if (b >= 0) {
        const int32_t slen = p.b_slen[b], clen = p.b_clen[b];
        size = LZ4BLOCK_HEADER + (lz4block_stored(clen, slen) ? slen : clen);
    }
    if (writer_tail(w, i)) size += LZ4BLOCK_HEADER;
    p.i_size[i] = size;
}

// one warp per item of [i0, i0 + n): its header (the checksum left 0 for the seal) and payload
__global__ void __launch_bounds__(128)
lz4block_writer_emit_kernel(const FrameWriterPlan w, uint32_t i0, uint32_t n)
{
    const uint32_t t = blockIdx.x * 4 + (threadIdx.x >> 5);
    if (t >= n) return;
    const FramePlan& p = w.p;
    const uint32_t i = i0 + t;
    const int32_t b = p.i_block[i];
    if (b < 0) return;                                                  // the end block alone
    const int lane = lane_id();
    const int32_t slen = p.b_slen[b], clen = p.b_clen[b];
    const bool stored = lz4block_stored(clen, slen);
    const int32_t sz = stored ? slen : clen;
    uint8_t* d = p.dst + writer_item_pos(w, i);
    if (lane < LZ4BLOCK_HEADER)
        d[lane] = lz4block_header_byte(lane, (stored ? LZ4BLOCK_RAW : LZ4BLOCK_LZ4) | p.level, (uint32_t)sz, (uint32_t)slen, 0);
    warp_copy(d + LZ4BLOCK_HEADER, stored ? p.src + p.b_soff[b] : p.slots + p.b_slot[b], sz, lane);
}

// one thread per item of the call, after every chunk and checksum
__global__ void __launch_bounds__(256)
lz4block_writer_seal_kernel(const FrameWriterPlan w)
{
    const FramePlan& p = w.p;
    const uint32_t i = blockIdx.x * 256 + threadIdx.x;
    if (i >= p.nitems) return;
    const uint32_t f = p.i_frame[i];
    const int32_t b = p.i_block[i];
    const uint64_t start = writer_item_pos(w, i), end = start + (uint64_t)p.i_size[i];
    if (b >= 0) put_le32(p.dst + start + 17, p.b_sum[b] & 0x0FFFFFFFu);   // the Checksum view keeps 28 bits
    if (writer_tail(w, i)) {                                            // finish(): the empty end block (:255-266)
        uint8_t* e = p.dst + end - LZ4BLOCK_HEADER;
        for (int k = 0; k < LZ4BLOCK_HEADER; k++) e[k] = lz4block_header_byte(k, LZ4BLOCK_RAW | p.level, 0, 0, 0);
    }
    if (item_last(p, i)) { p.f_off[f] = w.f_doff[f]; p.f_end[f] = end; }
}

// ---- incremental reader
// The counting walk's sink: how many blocks of each method the call takes (the walk applies the room).
struct Lz4BlockReaderCountSink {
    int32_t nc = 0, nr = 0;
    __device__ void block(uint64_t, bool raw, int32_t, int32_t, uint32_t) { (raw ? nr : nc)++; }
};

// The recording walk's sink: each block taken, at its place in d_dst (the stream's dst_off + the lengths before it), and
// where its unit starts in the piece.  c, qr, k: the stream's next compressed, stored and any record.
struct Lz4BlockReaderRecordSink {
    const Lz4BlockReaderRead& q; uint64_t soff, doff, c, qr, k;
    __device__ void block(uint64_t at, bool raw, int32_t clen, int32_t olen, uint32_t check)
    {
        const Lz4BlockRead& r = q.r;
        if (raw) { r.r_soff[qr] = soff + at; r.r_doff[qr] = doff; r.r_len[qr] = olen; qr++; }
        else { r.c_soff[c] = soff + at; r.c_doff[c] = doff; r.c_clen[c] = clen; r.c_olen[c] = olen; }
        r.b_doff[k] = doff; r.b_len[k] = olen; r.b_want[k] = check; r.b_comp[k] = raw ? -1 : (int32_t)c;
        q.k_at[k] = at - LZ4BLOCK_HEADER;
        if (!raw) c++;
        k++; doff += (uint64_t)olen;
    }
};

__global__ void __launch_bounds__(128)
lz4block_reader_walk_kernel(const Lz4BlockReaderRead q, bool record)
{
    const Lz4BlockRead& r = q.r;
    const uint32_t s = blockIdx.x * 128 + threadIdx.x;
    if (s >= r.ns) return;
    const int32_t latched = q.st_in[s];
    const uint8_t* src = r.src + r.s_off[s];
    const uint64_t n = r.s_len[s];
    const bool more = !q.eof[s];
    if (!record) {
        if (latched) {                                                  // DONE or an error: nothing is read
            r.n_comp[s] = 0; r.n_raw[s] = 0; r.tail[s] = latched; r.consumed[s] = 0; q.need[s] = 0;
            return;
        }
        Lz4BlockReaderCountSink sink;
        const Lz4BlockEnd e = walk_lz4block_from(src, n, r.stop, more, r.d_cap[s], sink);
        r.n_comp[s] = sink.nc; r.n_raw[s] = sink.nr;
        r.tail[s] = e.err ? e.err : e.stop == WALK_STOP_INPUT ? READER_MORE_INPUT : e.stop == WALK_STOP_ROOM ? READER_MORE_ROOM
                  : READER_DONE;
        r.consumed[s] = e.ip; q.need[s] = e.need;
        return;
    }
    if (latched) return;
    Lz4BlockReaderRecordSink sink{ q, r.s_off[s], r.d_off[s], r.p_comp[s], r.p_raw[s], r.p_comp[s] + r.p_raw[s] };
    walk_lz4block_from(src, n, r.stop, more, r.d_cap[s], sink);
}

// per block the reader decodes, compares the consumed length, then the checksum -- all "Stream is corrupted" (:236-262).  The
// blocks in front of the first failing one are delivered; the cut is where its unit starts.
__global__ void __launch_bounds__(128)
lz4block_reader_verdict_kernel(const Lz4BlockReaderRead q)
{
    const Lz4BlockRead& r = q.r;
    const uint32_t s = blockIdx.x * 4 + (threadIdx.x >> 5);
    if (s >= r.ns) return;
    const int lane = lane_id();
    const uint64_t k0 = r.p_comp[s] + r.p_raw[s], k1 = k0 + (uint64_t)r.n_comp[s] + (uint64_t)r.n_raw[s];
    uint64_t produced = 0, cut_at = 0;
    bool bad = false;
    for (uint64_t base = k0; base < k1; base += 32) {
        const uint64_t k = base + (uint64_t)lane;
        bool e = false;
        int32_t l = 0;
        if (k < k1) {
            const int32_t c = r.b_comp[k];
            e = (c >= 0 && r.c_res[c] != r.c_clen[c]) || (r.b_sum[k] & 0x0FFFFFFFu) != r.b_want[k];
            l = r.b_len[k];
        }
        const uint32_t m = __ballot_sync(B200_FULL, e);
        const int at = m ? __ffs((int)m) - 1 : 32;
        if (lane >= at) l = 0;
        for (int d = 16; d; d >>= 1) l += __shfl_xor_sync(B200_FULL, l, d);
        produced += (uint64_t)(uint32_t)l;
        if (m) { bad = true; cut_at = q.k_at[base + (uint64_t)at]; break; }
    }
    if (lane == 0) {
        const int32_t status = q.st_in[s] ? q.st_in[s] : bad ? -2 : r.tail[s];
        q.status[s] = status; q.produced[s] = produced;
        if (bad) r.consumed[s] = cut_at;
        if (status < 0 || status == READER_DONE) q.need[s] = 0;
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

cudaError_t launch_lz4block_writer_sizes(const FrameWriterPlan& w, uint32_t i0, uint32_t n, cudaStream_t st)
{
    if (n == 0) return cudaSuccess;
    B200_LAUNCH(lz4block_writer_size_kernel, (n + 255) / 256, 256, st, w, i0, n);
    return cudaGetLastError();
}
cudaError_t launch_lz4block_writer_emit(const FrameWriterPlan& w, uint32_t i0, uint32_t n, cudaStream_t st)
{
    if (n == 0) return cudaSuccess;
    B200_LAUNCH(lz4block_writer_emit_kernel, (n + 3) / 4, 128, st, w, i0, n);
    return cudaGetLastError();
}
cudaError_t launch_lz4block_writer_seal(const FrameWriterPlan& w, cudaStream_t st)
{
    if (w.p.nitems == 0) return cudaSuccess;
    B200_LAUNCH(lz4block_writer_seal_kernel, (w.p.nitems + 255) / 256, 256, st, w);
    return cudaGetLastError();
}
cudaError_t launch_lz4block_reader_walk(const Lz4BlockReaderRead& q, bool record, cudaStream_t st)
{
    if (q.r.ns == 0) return cudaSuccess;
    B200_LAUNCH(lz4block_reader_walk_kernel, (q.r.ns + 127) / 128, 128, st, q, record);
    return cudaGetLastError();
}
cudaError_t launch_lz4block_reader_verdict(const Lz4BlockReaderRead& q, cudaStream_t st)
{
    if (q.r.ns == 0) return cudaSuccess;
    B200_LAUNCH(lz4block_reader_verdict_kernel, (q.r.ns + 3) / 4, 128, st, q);
    return cudaGetLastError();
}

} // namespace b200
