// copy_count.h — TEST INFRASTRUCTURE ONLY.  Force-included (g++ -include) into every source of a counting variant of the
// emulator library, tests/simt/_build/libb200lz4_sim_counted.so, which tests/test_frame_decode_sim.py builds.  Every
// cudaMemcpyAsync the library's host layer makes then also adds its bytes to a counter per direction, which
// b200lz4_sim_copied_bytes (copy_count.cpp) reads: the tests check with it what crosses between host and device.  The
// product library and the plain emulator library (build_sim_library.sh) do not include it.
#pragma once
#include "simt.h"

namespace simt_count {
inline unsigned long long* bytes() { static unsigned long long c[2] = { 0, 0 }; return c; }    // host->device, device->host
static inline cudaError_t memcpy_async(void* d, const void* s, size_t n, cudaMemcpyKind k, cudaStream_t st = nullptr)
{
    if (k == cudaMemcpyHostToDevice) bytes()[0] += n;
    if (k == cudaMemcpyDeviceToHost) bytes()[1] += n;
    return cudaMemcpyAsync(d, s, n, k, st);
}
} // namespace simt_count

#define cudaMemcpyAsync simt_count::memcpy_async
