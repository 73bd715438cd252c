// tag_harness.cpp — the <= 64 KiB fast-compress kernel of lz4-java_b200/csrc at every hash-tag width, on the SIMT emulator
// (simt.h), exported with a C ABI for tests/test_compress_tags.py.  Test infrastructure only.
#include "../../lz4-java_b200/csrc/lz4_compress.cu"

using namespace b200;

#define ARGS src, &zero, &sl, dst, &zero, &dc, &res, 1u

template <int NW>
static void wide(const uint8_t* src, uint8_t* dst, uint64_t& zero, int32_t& sl, int32_t& dc, int32_t& res, int tag_bits)
{
    switch (tag_bits) {
    case 0: simt::launch(1, 32 * NW, [&] { lz4_compress_wide_kernel<13, 2, 2, NW, 1, 0>(ARGS); }); break;
    case 1: simt::launch(1, 32 * NW, [&] { lz4_compress_wide_kernel<13, 2, 2, NW, 1, 1>(ARGS); }); break;
    case 2: simt::launch(1, 32 * NW, [&] { lz4_compress_wide_kernel<13, 2, 2, NW, 1, 2>(ARGS); }); break;
    case 4: simt::launch(1, 32 * NW, [&] { lz4_compress_wide_kernel<13, 2, 2, NW, 1, 4>(ARGS); }); break;
    case 8: simt::launch(1, 32 * NW, [&] { lz4_compress_wide_kernel<13, 2, 2, NW, 1, 8>(ARGS); }); break;
    default: res = -1;
    }
}

// nw warps per block (3 or 2), tag_bits hash-tag bits per table slot (0, 1, 2, 4, 8)
extern "C" int sim_compress_wide(const uint8_t* src, int n, uint8_t* dst, int cap, int nw, int tag_bits)
{
    uint64_t zero = 0; int32_t sl = n, dc = cap, res = 0x7FFFFFFF;
    if (nw == 3) wide<3>(src, dst, zero, sl, dc, res, tag_bits);
    else wide<2>(src, dst, zero, sl, dc, res, tag_bits);
    return res;
}
#undef ARGS
