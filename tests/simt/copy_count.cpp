// copy_count.cpp — TEST INFRASTRUCTURE ONLY: the accessors of the counting emulator library (copy_count.h).
#include "copy_count.h"

// bytes the library has copied host->device and device->host so far
extern "C" void b200lz4_sim_copied_bytes(unsigned long long* h2d, unsigned long long* d2h)
{
    *h2d = simt_count::bytes()[0]; *d2h = simt_count::bytes()[1];
}

// the calling thread's current device in the stand-in runtime (what cudaGetDevice returns)
extern "C" int b200lz4_sim_current_device(void) { return simt_rt::current_device(); }
