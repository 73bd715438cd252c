// alloc_count.h — TEST INFRASTRUCTURE ONLY.  Force-included (g++ -include) into every source of the counting emulator library
// that tests/test_frame_reader_sim.py builds, in place of copy_count.h, which it includes: host<->device copies are counted as
// there, and every cudaMalloc / cudaFree the library makes also moves a count of live device bytes and its peak, which
// b200lz4_sim_device_bytes (alloc_count.cpp) reads.  The tests check with it what device memory a call keeps.  The product
// library and the other emulator libraries do not include it.
#pragma once
#include "copy_count.h"
#include <map>
#include <mutex>

namespace simt_count {
// live device bytes and their peak since the last reset, under one lock (calls may come from several threads)
struct DeviceBytes { std::mutex m; std::map<void*, size_t> size; unsigned long long live = 0, peak = 0; };
inline DeviceBytes& device_bytes() { static DeviceBytes d; return d; }
template <class T> static inline cudaError_t malloc_counted(T** p, size_t n)
{
    const cudaError_t e = cudaMalloc(p, n);
    if (e == cudaSuccess) {
        DeviceBytes& d = device_bytes(); std::lock_guard<std::mutex> g(d.m);
        d.size[(void*)*p] = n; d.live += n; if (d.live > d.peak) d.peak = d.live;
    }
    return e;
}
static inline cudaError_t free_counted(void* p)
{
    {
        DeviceBytes& d = device_bytes(); std::lock_guard<std::mutex> g(d.m);
        auto it = d.size.find(p);
        if (it != d.size.end()) { d.live -= it->second; d.size.erase(it); }
    }
    return cudaFree(p);
}
} // namespace simt_count

#define cudaMalloc simt_count::malloc_counted
#define cudaFree simt_count::free_counted
