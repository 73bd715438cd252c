// copy_count.cpp — TEST INFRASTRUCTURE ONLY: the accessor of the counting emulator library (copy_count.h).
#include "copy_count.h"

// bytes the library has copied host->device and device->host so far
extern "C" void b200lz4_sim_copied_bytes(unsigned long long* h2d, unsigned long long* d2h)
{
    *h2d = simt_count::bytes()[0]; *d2h = simt_count::bytes()[1];
}
