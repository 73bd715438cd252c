// kernels.h — internal launch interface between the C-ABI layer (capi.cu) and the kernels.
#pragma once
#include <atomic>
#include <cstddef>
#include <cstdint>
#ifdef B200_HOST_SIM
#include "simt.h"
#else
#include <cuda_runtime.h>
#endif

namespace b200 {

// One batch of independent LZ4 blocks (or hash buffers); every pointer is a device pointer.
struct BatchArgs {
    const uint8_t*  src_base;
    const uint64_t* src_off;
    const int32_t*  src_len;    // compress: bytes to compress; safe: compressed size; fast: readable bytes
    uint8_t*        dst_base;
    const uint64_t* dst_off;
    const int32_t*  dst_cap;    // compress/safe: capacity; fast: exact decoded size
    int32_t*        result;
    size_t          n;
};

cudaError_t launch_decompress_safe(const BatchArgs& a, cudaStream_t st);
cudaError_t launch_decompress_fast(const BatchArgs& a, cudaStream_t st);
cudaError_t launch_compress_fast(const BatchArgs& a, int max_src_len, cudaStream_t st);
cudaError_t launch_compress_hc(const BatchArgs& a, int level, cudaStream_t st);
cudaError_t launch_xxh32(const uint8_t* base, const uint64_t* off, const int32_t* len, uint32_t seed,
                         uint32_t* out, size_t n, cudaStream_t st);
// One warp per buffer: for a few long streams (frame content checksums).
cudaError_t launch_xxh32_long(const uint8_t* base, const uint64_t* off, const int32_t* len, uint32_t seed,
                              uint32_t* out, size_t n, cudaStream_t st);
// frame content checksums chained to the block decoder (frame.cu): one warp per frame follows the decoder's result words
static constexpr int32_t FRAME_RES_PENDING = int32_t(0x80808080);      // what cudaMemset(0x80) leaves; no decoder result looks like it
cudaError_t launch_xxh32_frames_chained(const uint8_t* slots, const uint64_t* blk_off, const uint32_t* f_first, const uint32_t* f_nblk,
                                        const int32_t* blk_comp, const int32_t* blk_rawlen, const int32_t* c_res,
                                        uint32_t* out, size_t n, cudaStream_t st);
cudaError_t launch_xxh64(const uint8_t* base, const uint64_t* off, const int32_t* len, uint64_t seed,
                         uint64_t* out, size_t n, cudaStream_t st);

// streaming hash: one device-resident state per handle, updated by a single-warp kernel
struct Xxh32State { uint64_t total; uint32_t v[4]; uint8_t mem[16]; uint32_t memsize; uint32_t seed; uint32_t digest; };
struct Xxh64State { uint64_t total; uint64_t v[4]; uint8_t mem[32]; uint32_t memsize; uint32_t pad; uint64_t seed; uint64_t digest; };
cudaError_t launch_xxh32_stream(Xxh32State* st, int op, uint32_t seed, const uint8_t* data, size_t len, cudaStream_t s);
cudaError_t launch_xxh64_stream(Xxh64State* st, int op, uint64_t seed, const uint8_t* data, size_t len, cudaStream_t s);
enum { XXH_OP_RESET = 0, XXH_OP_UPDATE = 1, XXH_OP_DIGEST = 2 };

cudaError_t launch_xxh64_long(const uint8_t* base, const uint64_t* off, const int32_t* len, uint64_t seed,
                              uint64_t* out, size_t n, cudaStream_t st);

// prefix-sum compaction of variable-length outputs (compact_host path)
cudaError_t launch_compact(const uint8_t* slots, const uint64_t* slot_off, const int32_t* lens,
                           uint8_t* out, uint64_t* out_off, uint64_t* total, size_t n, cudaStream_t st);
// the scan alone: out_off[i] = *carry_in + exclusive prefix of max(lens, 0); *total = *carry_in + the sum (carry_in may be
// NULL: 0).  carry_in and total must be different words.
cudaError_t launch_scan(const int32_t* lens, uint64_t* out_off, uint64_t* total, const uint64_t* carry_in, size_t n, cudaStream_t st);

// ---- device-resident LZ4 Frame writer (frame_encode.cu, driven by b200lz4f_compress_dev in containers.cu)
// The frame descriptor LZ4FrameOutputStream.writeHeader puts between the magic and the header checksum byte
// (LZ4FrameOutputStream.java:178-187): FLG, BD and, with flags bit 2, the 8-byte content size.  flags: bit0 content
// checksum, bit1 block checksums, bit2 content size.  Returns the bytes written, 2 or 10.  Both frame writers call it.
__host__ __device__ inline int frame_descriptor(uint8_t* d, int bsCode, int flags, uint64_t content_size)
{
    d[0] = (uint8_t)((1 << 6) | (1 << 5) | ((flags & 2) ? 1 << 4 : 0) | ((flags & 4) ? 1 << 3 : 0) | ((flags & 1) ? 1 << 2 : 0));
    d[1] = (uint8_t)(bsCode << 4);
    if (!(flags & 4)) return 2;
    for (int k = 0; k < 8; k++) d[2 + k] = (uint8_t)(content_size >> (8 * k));
    return 10;
}

// One call's descriptors, all device pointers.  An "item" is one block of a frame, or an empty frame (no block): the frame
// header rides on a frame's first item, the EndMark and content checksum on its last, so one scan of the item sizes places
// everything.  Items of a frame are consecutive; a frame's first / last item is where i_frame changes.
struct FramePlan {
    const uint8_t* src; uint8_t* dst; const uint8_t* slots;         // sources, the frames, one chunk's compressed blocks
    const uint64_t* b_soff; const int32_t* b_slen;                  // per block: source bytes
    const uint64_t* b_slot; const int32_t* b_clen;                  //   its slot in `slots` and the compressor's result
    uint64_t* b_poff; int32_t* b_plen; const uint32_t* b_sum;       //   the payload as written, and its XXH32 (flags bit 1)
    const uint32_t* i_frame; const int32_t* i_block;                // per item: frame, block (-1: an empty frame)
    int32_t* i_size; uint64_t* i_off;                               //   bytes it takes, where it starts in dst
    const uint64_t* f_len; const uint32_t* f_sum;                   // per frame: content size, content checksum (flags bit 0)
    uint64_t* f_off; uint64_t* f_end;                               //   where it starts and ends in dst
    uint32_t nitems; int bsCode; int flags;
};
// items [i0, i0 + n): their sizes (frame_size_kernel), and their block words and payloads (frame_emit_kernel, one warp each)
cudaError_t launch_frame_sizes(const FramePlan& p, uint32_t i0, uint32_t n, cudaStream_t st);
cudaError_t launch_frame_emit(const FramePlan& p, uint32_t i0, uint32_t n, cudaStream_t st);
// every item: headers, block checksums, EndMarks, content checksums, f_off / f_end (frame_seal_kernel)
cudaError_t launch_frame_seal(const FramePlan& p, cudaStream_t st);

// Average buffer length from which the hash batches give each buffer a whole warp (launch_xxh*_long) instead of a lane.
static constexpr uint64_t XXH_LONG_AVG = 32768;

// LZ4_compressBound(len) (lz4.h:212) without its range check, and the room one block takes in a packed compress
// staging area: that bound rounded up to 16 bytes.
static inline uint64_t compress_bound(uint64_t len) { return len + len / 255 + 16; }
static inline uint64_t aligned_compress_bound(uint64_t len) { return (compress_bound(len) + 15) & ~uint64_t(15); }

extern std::atomic<unsigned long long> g_launch_count;      // every kernel launch the library makes (any thread): b200lz4_launch_count()

// ---- host layer shared by capi.cu and containers.cu
extern const size_t CHUNK_SPAN;                            // bytes of source per chunk of a chunked call (B200LZ4_CHUNK_MB, default 256)
static constexpr size_t CHUNK_BLOCKS = 1 << 16;            // blocks per chunk at most
int fail_arg(const char* what);                            // set the thread's error message, return B200LZ4_E_ARG
int fail_cuda(cudaError_t e, const char* where);           // ... B200LZ4_E_CUDA or _NODEVICE
int reserve_device(uint8_t*& p, size_t& cap, size_t need, int slack_shift = 2);   // grow-or-keep device buffer
int reserve_pinned(uint8_t*& p, size_t& cap, size_t need);                       // grow-or-keep pinned buffer
// Grow-or-keep scratch of b200lz4f_compress_dev, one per thread and device (it lives in the thread's context).
struct FrameScratch {
    uint8_t* d_plan = nullptr; size_t plan_cap = 0;        // the call's descriptors (FramePlan)
    uint8_t* h_plan = nullptr; size_t h_plan_cap = 0;      // pinned: their upload, and the results coming back
    uint8_t* d_slots = nullptr; size_t slots_cap = 0;      // one chunk's compressed blocks, bound-sized slots
    cudaStream_t st2 = nullptr; cudaEvent_t fork = nullptr, join = nullptr;   // content checksums run beside the rest
};
int get_frame_scratch(FrameScratch** out);                 // selects the thread's device, like every entry point

} // namespace b200
