// alloc_count.cpp — TEST INFRASTRUCTURE ONLY: the accessors of alloc_count.h's device-byte count.
#include "alloc_count.h"

// live device bytes, and the most there were since the last b200lz4_sim_reset_device_peak
extern "C" void b200lz4_sim_device_bytes(unsigned long long* live, unsigned long long* peak)
{
    simt_count::DeviceBytes& d = simt_count::device_bytes(); std::lock_guard<std::mutex> g(d.m);
    *live = d.live; *peak = d.peak;
}
extern "C" void b200lz4_sim_reset_device_peak(void)
{
    simt_count::DeviceBytes& d = simt_count::device_bytes(); std::lock_guard<std::mutex> g(d.m);
    d.peak = d.live;
}
