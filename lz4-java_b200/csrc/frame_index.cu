// frame_index.cu — the device half of the LZ4 Frame indexer b200lz4f_index_create_dev (frame.cu): the container walk of
// walk_frames (kernels.h) over bytes in device memory, so that only per-frame and per-block facts cross to the host.
//   frame_walk_kernel    one thread per segment [seg_start, seg_end): walks frames from seg_start until the first frame
//                        boundary at or past seg_end, writing 16-byte records into a region of its own
//   compact_scan_kernel  where each walker's records go when packed (launch_scan, compact.cu)
//   frame_pack_kernel    one CTA per walker: its records, back to back, for one copy to the host
// The walk is a chain of dependent loads (each block word says where the next one is), so one thread per segment is all
// the parallelism there is; segments come from the caller's hints at frame starts.
#include "common.cuh"
#include "kernels.h"

namespace b200 {

// The device sink of walk_frames: records in stream order into [recs, recs + cap); past cap it only counts.
struct RecordSink {
    WalkRec* recs; uint64_t cap, n = 0, frame_at = 0;
    __device__ void put(uint64_t at, uint64_t a, uint64_t b) { if (at < cap) { recs[at].a = a; recs[at].b = b; } }
    __device__ void frame_begin(const WalkFrame&) { frame_at = n; n += 2; }
    __device__ void block(uint64_t src_off, uint32_t word, uint32_t checksum) { put(n++, src_off, (uint64_t)word | ((uint64_t)checksum << 32)); }
    __device__ void frame_end(const WalkFrame& f)
    {
        // {desc_off, content_size}, {nblocks, content_checksum | flg | bd | hc_byte | desc_len and the three flags}
        const uint32_t bits = (uint32_t)f.flg | ((uint32_t)f.bd << 8) | ((uint32_t)f.hc_byte << 16) | ((uint32_t)(f.desc_len & 15) << 24) |
                              (f.complete ? 1u << 28 : 0u) | (f.has_checksum ? 1u << 29 : 0u) | (f.has_size ? 1u << 30 : 0u);
        put(frame_at, f.desc_off, f.content_size);
        put(frame_at + 1, f.nblocks, (uint64_t)f.content_checksum | ((uint64_t)bits << 32));
    }
};

__global__ void __launch_bounds__(128)
frame_walk_kernel(const uint8_t* src, uint64_t n, bool single, const WalkSeg* segs, WalkSummary* sum, int32_t* lens, WalkRec* recs, uint32_t m)
{
    const uint32_t j = blockIdx.x * 128 + threadIdx.x;
    if (j >= m) return;
    const WalkSeg s = segs[j];
    RecordSink sink{ recs + s.rec_off, s.rec_cap };
    const WalkEnd e = walk_frames(src, n, s.start, s.end, single, sink);
    sum[j] = WalkSummary{ e.ip, sink.n, e.err, (e.seen ? (uint32_t)WALK_SEEN : 0u) | (e.single_done ? (uint32_t)WALK_SINGLE_DONE : 0u) };
    lens[j] = (int32_t)(sink.n < s.rec_cap ? sink.n : s.rec_cap);
}

__global__ void __launch_bounds__(128)
frame_pack_kernel(const WalkSeg* segs, const int32_t* lens, const uint64_t* pos, const WalkRec* recs, WalkRec* packed)
{
    const uint32_t j = blockIdx.x;
    const WalkRec* from = recs + segs[j].rec_off;
    WalkRec* to = packed + pos[j];
    for (int32_t i = threadIdx.x; i < lens[j]; i += 128) to[i] = from[i];
}

// launchers: the same code in the emulator build (B200_LAUNCH)
cudaError_t launch_frame_walk(const uint8_t* src, uint64_t n, bool single, const WalkSeg* segs, WalkSummary* sum, int32_t* lens,
                              WalkRec* recs, uint32_t m, cudaStream_t st)
{
    if (m == 0) return cudaSuccess;
    B200_LAUNCH(frame_walk_kernel, (m + 127) / 128, 128, st, src, n, single, segs, sum, lens, recs, m);
    return cudaGetLastError();
}
cudaError_t launch_frame_pack(const WalkSeg* segs, const int32_t* lens, const uint64_t* pos, const WalkRec* recs, WalkRec* packed,
                              uint32_t m, cudaStream_t st)
{
    if (m == 0) return cudaSuccess;
    B200_LAUNCH(frame_pack_kernel, m, 128, st, segs, lens, pos, recs, packed);
    return cudaGetLastError();
}

} // namespace b200
