// compact.cu — device-side compaction of variable-length compressed blocks (SURVEY.md §8e "optional
// compaction = exclusive scan of lengths + gather"): blocks compressed into bound-sized slots are
// packed back-to-back so only real bytes cross PCIe on the way back to the host.
#include "common.cuh"
#include "kernels.h"

namespace b200 {

// exclusive scan of max(lens[i],0) over n <= ~10^5 entries by one CTA; writes out_off[] and *total.  carry_in (a device
// word, not `total`): where the scan starts, so a call cut into chunks carries its running offset from one chunk's scan to
// the next without the host; NULL starts at 0.
__global__ void __launch_bounds__(1024)
compact_scan_kernel(const int32_t* __restrict__ lens, uint64_t* __restrict__ out_off, uint64_t* __restrict__ total, uint32_t n,
                    const uint64_t* __restrict__ carry_in = nullptr)
{
    __shared__ uint64_t warp_sum[32];
    __shared__ uint64_t carry;
    const int lane = lane_id(), warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) carry = carry_in ? *carry_in : 0;
    __syncthreads();
    for (uint32_t base = 0; base < n; base += 1024) {
        const uint32_t i = base + threadIdx.x;
        const uint64_t v = i < n ? (uint64_t)max(lens[i], 0) : 0;
        uint64_t x = v;
        for (int d = 1; d < 32; d <<= 1) { const uint64_t y = __shfl_up_sync(B200_FULL, x, d); if (lane >= d) x += y; }
        if (lane == 31) warp_sum[warp] = x;
        __syncthreads();
        if (warp == 0) {
            uint64_t w = warp_sum[lane], s = w;
            for (int d = 1; d < 32; d <<= 1) { const uint64_t y = __shfl_up_sync(B200_FULL, s, d); if (lane >= d) s += y; }
            warp_sum[lane] = s - w;                       // exclusive prefix of the warp totals
        }
        __syncthreads();
        const uint64_t c = carry;
        if (i < n) out_off[i] = c + warp_sum[warp] + x - v;
        __syncthreads();
        if (threadIdx.x == 1023) carry = c + warp_sum[31] + x;
        __syncthreads();
    }
    if (threadIdx.x == 0) *total = carry;
}

// one warp per block: copy its bytes from the slot to the packed position
__global__ void __launch_bounds__(128)
compact_gather_kernel(const uint8_t* __restrict__ slots, const uint64_t* __restrict__ slot_off, const int32_t* __restrict__ lens,
                      uint8_t* __restrict__ out, const uint64_t* __restrict__ out_off, uint32_t n)
{
    const uint32_t b = blockIdx.x * 4 + (threadIdx.x >> 5);
    if (b >= n) return;
    const int len = lens[b];
    if (len > 0) warp_copy(out + out_off[b], slots + slot_off[b], len, lane_id());
}

// (the emulator build runs this one too: the device frame writer calls it)
cudaError_t launch_scan(const int32_t* lens, uint64_t* out_off, uint64_t* total, const uint64_t* carry_in, size_t n, cudaStream_t st)
{
    B200_LAUNCH(compact_scan_kernel, 1, 1024, st, lens, out_off, total, (uint32_t)n, carry_in);
    return cudaGetLastError();
}

#ifndef B200_HOST_SIM          // launchers: CUDA only
cudaError_t launch_compact(const uint8_t* slots, const uint64_t* slot_off, const int32_t* lens,
                           uint8_t* out, uint64_t* out_off, uint64_t* total, size_t n, cudaStream_t st)
{
    if (n == 0) return cudaSuccess;
    compact_scan_kernel<<<1, 1024, 0, st>>>(lens, out_off, total, (uint32_t)n);
    cudaError_t e = cudaGetLastError(); if (e != cudaSuccess) return e;
    compact_gather_kernel<<<(unsigned)((n + 3) / 4), 128, 0, st>>>(slots, slot_off, lens, out, out_off, (uint32_t)n);
    return cudaGetLastError();
}

cudaError_t launch_gather(const uint8_t* src, const uint64_t* src_off, const int32_t* lens,
                          uint8_t* dst, const uint64_t* dst_off, size_t n, cudaStream_t st)
{
    if (n == 0) return cudaSuccess;
    compact_gather_kernel<<<(unsigned)((n + 3) / 4), 128, 0, st>>>(src, src_off, lens, dst, dst_off, (uint32_t)n);
    return cudaGetLastError();
}

#endif

} // namespace b200
