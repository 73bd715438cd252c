// simt.h — a small single-threaded SIMT emulator (TEST INFRASTRUCTURE ONLY).
//
// Purpose: run the *same source* of the CUDA kernels in lz4-java_b200/csrc on the CPU, so their control logic
// (token walks, margins, dependency rounds, producer/consumer hand-offs) can be fuzzed against the oracle on the
// build box, which has no GPU.  A kernel source is compiled as host C++ with -DB200_HOST_SIM, which makes
// common.cuh include this header instead of <cuda_runtime.h>.  Nothing in the product ever includes it, and it
// is not a fallback: it exists under tests/ and is driven only by tests/test_kernel_logic_cpu.py.
//
// Model: every CUDA thread of ONE CTA is a ucontext coroutine on one OS thread.  A thread runs until it reaches a
// warp collective (__shfl*_sync, __ballot_sync, __syncwarp, ...) or a CTA barrier (__syncthreads, bar.sync /
// bar.arrive with an id and a thread count); then the scheduler runs the next one.  A warp collective completes
// when every not-yet-exited thread of the warp has reached it — the emulator aborts if they reached different
// call sites (divergent full-mask collectives are undefined behaviour on the GPU) or if nothing can make progress
// (deadlock).  Memory is host memory: plain loads/stores, atomics are ordinary read-modify-writes.  What this
// checks is logic, not timing and not memory-model subtleties.
#pragma once
#include <cstdint>
#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>
#include <functional>
#include <algorithm>
#include <mutex>
#include <ucontext.h>

// ---- CUDA spellings
#define __device__
#define __host__
#define __global__
#define __forceinline__ inline __attribute__((always_inline))
#define __launch_bounds__(...)
#define __restrict__ __restrict
#define __shared__ static
#define __align__(n) __attribute__((aligned(n)))
typedef int cudaError_t;
typedef void* cudaStream_t;
typedef void* cudaEvent_t;
enum { cudaSuccess = 0, cudaErrorNoDevice = 100, cudaErrorInsufficientDriver = 35, cudaErrorInitializationError = 3 };
enum cudaMemcpyKind { cudaMemcpyHostToHost, cudaMemcpyHostToDevice, cudaMemcpyDeviceToHost, cudaMemcpyDeviceToDevice, cudaMemcpyDefault };
enum { cudaStreamNonBlocking = 1, cudaHostAllocDefault = 0, cudaEventDisableTiming = 2, cudaHostRegisterPortable = 1 };

// ---- a stand-in for the slice of the CUDA runtime that the library's host layer (capi.cu, frame.cu) calls, so the whole
// library can be built for the emulator (tests/simt/build_sim_library.sh).  Everything is synchronous; "device memory" is
// host heap with 256-byte guard bands (the kernels read the aligned words around their buffers).
namespace simt_rt {
inline void* alloc(size_t n) { char* raw = (char*)std::calloc(n + 768, 1); if (!raw) return nullptr; char* p = raw + 256 + ((256 - ((uintptr_t)(raw + 256) & 255)) & 255); ((void**)p)[-1] = raw; return p; }
inline void release(void* p) { if (p) std::free(((void**)p)[-1]); }
}
template <class T> static inline cudaError_t cudaMalloc(T** p, size_t n) { *p = (T*)simt_rt::alloc(n); return *p ? cudaSuccess : 2; }
static inline cudaError_t cudaFree(void* p) { simt_rt::release(p); return cudaSuccess; }
// SIMT_FAIL_HOST_ALLOC set: every pinned allocation fails, as a real one can when the host is short of pinnable memory
template <class T> static inline cudaError_t cudaHostAlloc(T** p, size_t n, unsigned)
{ *p = std::getenv("SIMT_FAIL_HOST_ALLOC") ? nullptr : (T*)simt_rt::alloc(n); return *p ? cudaSuccess : 2; }
static inline cudaError_t cudaFreeHost(void* p) { simt_rt::release(p); return cudaSuccess; }
static inline cudaError_t cudaHostRegister(void*, size_t, unsigned) { return cudaSuccess; }
static inline cudaError_t cudaHostUnregister(void*) { return cudaSuccess; }
static inline cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, cudaMemcpyKind, cudaStream_t = nullptr) { if (n) std::memmove(d, s, n); return cudaSuccess; }
static inline cudaError_t cudaMemsetAsync(void* d, int v, size_t n, cudaStream_t = nullptr) { std::memset(d, v, n); return cudaSuccess; }
namespace simt_rt {
inline int device_count() { const char* e = std::getenv("SIMT_DEVICES"); int n = e ? std::atoi(e) : 1; return n < 1 ? 1 : n; }   // pretend GPUs (multi-device host logic)
inline int& current_device() { static thread_local int d = 0; return d; }
}
static inline cudaError_t cudaGetDeviceCount(int* n) { *n = simt_rt::device_count(); return cudaSuccess; }
static inline cudaError_t cudaSetDevice(int d) { if (d < 0 || d >= simt_rt::device_count()) return 101; simt_rt::current_device() = d; return cudaSuccess; }
static inline cudaError_t cudaDeviceCanAccessPeer(int* can, int a, int b) { *can = a != b; return cudaSuccess; }
static inline cudaError_t cudaDeviceEnablePeerAccess(int, unsigned) { return cudaSuccess; }
static inline cudaError_t cudaMemcpyPeerAsync(void* d, int, const void* s, int, size_t n, cudaStream_t = nullptr) { if (n) std::memmove(d, s, n); return cudaSuccess; }
static inline cudaError_t cudaGetDevice(int* d) { *d = simt_rt::current_device(); return cudaSuccess; }
static inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t* s, unsigned) { *s = std::malloc(8); return cudaSuccess; }
static inline cudaError_t cudaStreamDestroy(cudaStream_t s) { std::free(s); return cudaSuccess; }
static inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
static inline cudaError_t cudaEventCreateWithFlags(cudaEvent_t* e, unsigned) { *e = std::malloc(8); return cudaSuccess; }
static inline cudaError_t cudaEventDestroy(cudaEvent_t e) { std::free(e); return cudaSuccess; }
static inline cudaError_t cudaEventRecord(cudaEvent_t, cudaStream_t = nullptr) { return cudaSuccess; }
static inline cudaError_t cudaEventSynchronize(cudaEvent_t) { return cudaSuccess; }
static inline cudaError_t cudaStreamWaitEvent(cudaStream_t, cudaEvent_t, unsigned = 0) { return cudaSuccess; }
static inline cudaError_t cudaGetLastError() { return cudaSuccess; }
static inline const char* cudaGetErrorString(cudaError_t) { return "simt emulator"; }

struct uint2 { uint32_t x, y; };
struct uint4 { uint32_t x, y, z, w; };
static inline uint2 make_uint2(uint32_t x, uint32_t y) { return uint2{x, y}; }
static inline uint4 make_uint4(uint32_t x, uint32_t y, uint32_t z, uint32_t w) { return uint4{x, y, z, w}; }

// CUDA's mixed-type min/max overloads
static inline int min(int a, int b) { return a < b ? a : b; }
static inline int max(int a, int b) { return a > b ? a : b; }
static inline unsigned min(unsigned a, unsigned b) { return a < b ? a : b; }
static inline unsigned max(unsigned a, unsigned b) { return a > b ? a : b; }
static inline unsigned min(unsigned a, int b) { return min(a, (unsigned)b); }
static inline unsigned min(int a, unsigned b) { return min((unsigned)a, b); }
static inline unsigned max(unsigned a, int b) { return max(a, (unsigned)b); }
static inline unsigned max(int a, unsigned b) { return max((unsigned)a, b); }
static inline long long min(long long a, long long b) { return a < b ? a : b; }
static inline long long max(long long a, long long b) { return a > b ? a : b; }
static inline unsigned long long min(unsigned long long a, unsigned long long b) { return a < b ? a : b; }
static inline unsigned long long max(unsigned long long a, unsigned long long b) { return a > b ? a : b; }
static inline unsigned long min(unsigned long a, unsigned long b) { return a < b ? a : b; }
static inline unsigned long max(unsigned long a, unsigned long b) { return a > b ? a : b; }

static inline int __ffs(int x) { return x ? __builtin_ctz((unsigned)x) + 1 : 0; }
static inline int __clz(int x) { return x ? __builtin_clz((unsigned)x) : 32; }
static inline unsigned __brev(unsigned x) { unsigned r = 0; for (int i = 0; i < 32; i++) if (x & (1u << i)) r |= 1u << (31 - i); return r; }
static inline int __popc(unsigned x) { return __builtin_popcount(x); }
static inline int __ffsll(long long x) { return x ? __builtin_ctzll((unsigned long long)x) + 1 : 0; }
static inline int __clzll(long long x) { return x ? __builtin_clzll((unsigned long long)x) : 64; }
static inline int __popcll(unsigned long long x) { return __builtin_popcountll(x); }
static inline uint32_t __funnelshift_r(uint32_t lo, uint32_t hi, uint32_t s) { return (uint32_t)((((uint64_t)hi << 32) | lo) >> (s & 31)); }
static inline uint32_t __byte_perm(uint32_t x, uint32_t y, uint32_t s) { const uint64_t v = ((uint64_t)y << 32) | x; uint32_t r = 0; for (int i = 0; i < 4; i++) { const uint32_t sel = (s >> (4 * i)) & 15u; uint32_t b = (uint32_t)(v >> (8 * (sel & 7u))) & 0xFFu; if (sel & 8u) b = (b & 0x80u) ? 0xFFu : 0u; r |= b << (8 * i); } return r; }
static inline uint32_t __funnelshift_rc(uint32_t lo, uint32_t hi, uint32_t s) { return (uint32_t)((((uint64_t)hi << 32) | lo) >> (s > 32 ? 32 : s)); }
static inline uint32_t __funnelshift_l(uint32_t lo, uint32_t hi, uint32_t s) { return (uint32_t)(((((uint64_t)hi << 32) | lo) << (s & 31)) >> 32); }
static inline size_t __cvta_generic_to_shared(const void* p) { return (size_t)p; }
static inline size_t __cvta_generic_to_global(const void* p) { return (size_t)p; }
static inline void __threadfence_block() {}
static inline void __threadfence() {}
static inline unsigned atomicAdd(unsigned* p, unsigned v) { unsigned o = *p; *p = o + v; return o; }
static inline int atomicAdd(int* p, int v) { int o = *p; *p = o + v; return o; }

namespace simt {

struct Idx { unsigned x, y, z; };
enum OpKind { OP_NONE, OP_SHFL, OP_BALLOT, OP_SYNCWARP, OP_REDUCE_MAX, OP_REDUCE_OR, OP_MATCH_ANY };
enum State { ST_RUN, ST_WARP_OP, ST_BAR_WAIT, ST_DONE };

struct Lane {
    ucontext_t ctx;
    std::vector<char> stack;
    int tid = 0;
    State st = ST_RUN;
    int op_kind = OP_NONE, op_line = 0, op_src = 0;
    uint32_t op_val = 0, op_res = 0;
    int bar_id = -1;
};
struct Barrier { int arrived = 0; };

struct Cta {
    std::vector<Lane> lanes;
    Barrier bars[16];
    Idx block{0, 0, 0}, dim{1, 1, 1}, grid{1, 1, 1};
    std::function<void()> body;
};

inline Cta*& cta() { static Cta* c = nullptr; return c; }
inline uint8_t* dyn_smem() { alignas(128) static uint8_t mem[232448]; return mem; }     // the CTA's dynamic shared memory
inline Lane*& cur() { static Lane* l = nullptr; return l; }
inline ucontext_t& sched_ctx() { static ucontext_t c; return c; }

[[noreturn]] inline void die(const char* what, int a = 0, int b = 0)
{
    std::fprintf(stderr, "simt: %s (%d, %d)\n", what, a, b);
    std::abort();
}

inline void yield() { swapcontext(&cur()->ctx, &sched_ctx()); }

inline uint32_t warp_op(int kind, int line, uint32_t val, int src)
{
    Lane* l = cur();
    l->st = ST_WARP_OP; l->op_kind = kind; l->op_line = line; l->op_val = val; l->op_src = src;
    yield();
    return l->op_res;
}

inline void release_barrier(int id)
{
    Cta* c = cta();
    c->bars[id].arrived = 0;
    for (Lane& l : c->lanes) if (l.st == ST_BAR_WAIT && l.bar_id == id) { l.st = ST_RUN; l.bar_id = -1; }
}
inline void bar_arrive(int id, int count)
{
    Barrier& b = cta()->bars[id];
    if (++b.arrived == count) release_barrier(id);
    else if (b.arrived > count) die("barrier over-arrival", id, b.arrived);
}
inline void bar_sync(int id, int count)
{
    Lane* l = cur();
    Barrier& b = cta()->bars[id];
    l->st = ST_BAR_WAIT; l->bar_id = id;
    if (++b.arrived == count) { release_barrier(id); return; }
    if (b.arrived > count) die("barrier over-arrival", id, b.arrived);
    yield();
}

inline void complete_warp(Lane* w, int n)            // all live lanes of this warp wait at a collective
{
    int kind = -1, line = -1;
    for (int i = 0; i < n; i++) {
        if (w[i].st != ST_WARP_OP) continue;
        if (kind < 0) { kind = w[i].op_kind; line = w[i].op_line; }
        else if (w[i].op_kind != kind || w[i].op_line != line) die("divergent warp collective: source lines", line, w[i].op_line);
    }
    uint32_t ballot = 0, rmax = 0, ror = 0; bool first = true;
    for (int i = 0; i < n; i++) if (w[i].st == ST_WARP_OP) {
        if (w[i].op_val) ballot |= 1u << i;
        ror |= w[i].op_val;
        if (first || (int32_t)w[i].op_val > (int32_t)rmax) { rmax = w[i].op_val; first = false; }
    }
    for (int i = 0; i < n; i++) {
        if (w[i].st != ST_WARP_OP) continue;
        switch (kind) {
        case OP_SHFL: { const int s = w[i].op_src; w[i].op_res = (s >= 0 && s < n && w[s].st == ST_WARP_OP) ? w[s].op_val : w[i].op_val; break; }
        case OP_BALLOT: w[i].op_res = ballot; break;
        case OP_REDUCE_MAX: w[i].op_res = rmax; break;
        case OP_REDUCE_OR: w[i].op_res = ror; break;
        case OP_MATCH_ANY: { uint32_t m = 0; for (int j = 0; j < n; j++) if (w[j].st == ST_WARP_OP && w[j].op_val == w[i].op_val) m |= 1u << j; w[i].op_res = m; break; }
        default: w[i].op_res = 0; break;
        }
    }
    for (int i = 0; i < n; i++) if (w[i].st == ST_WARP_OP) w[i].st = ST_RUN;
}

inline void lane_entry()
{
    cta()->body();
    cur()->st = ST_DONE;
    swapcontext(&cur()->ctx, &sched_ctx());
}

// Run one CTA of `nthreads` threads to completion.
inline void run_cta(int nthreads, Idx block, Idx grid, std::function<void()> body)
{
    Cta c; c.block = block; c.grid = grid; c.dim = Idx{(unsigned)nthreads, 1, 1}; c.body = std::move(body);
    c.lanes.resize(nthreads);
    cta() = &c;
    for (int t = 0; t < nthreads; t++) {
        Lane& l = c.lanes[t];
        l.tid = t; l.stack.resize(256 * 1024);
        getcontext(&l.ctx);
        l.ctx.uc_stack.ss_sp = l.stack.data(); l.ctx.uc_stack.ss_size = l.stack.size(); l.ctx.uc_link = nullptr;
        makecontext(&l.ctx, (void (*)())lane_entry, 0);
    }
    for (;;) {
        bool progressed = false, alive = false;
        for (Lane& l : c.lanes) {
            if (l.st == ST_RUN) { cur() = &l; swapcontext(&sched_ctx(), &l.ctx); progressed = true; }
            if (l.st != ST_DONE) alive = true;
        }
        if (!alive) break;
        for (int w0 = 0; w0 < nthreads; w0 += 32) {
            const int n = std::min(32, nthreads - w0);
            bool any = false, all = true;
            for (int i = 0; i < n; i++) { const State s = c.lanes[w0 + i].st; if (s == ST_WARP_OP) any = true; else if (s != ST_DONE) all = false; }
            if (any && all) { complete_warp(&c.lanes[w0], n); progressed = true; }
        }
        if (!progressed) {
            for (Lane& l : c.lanes) std::fprintf(stderr, "  tid %d state %d line %d bar %d\n", l.tid, (int)l.st, l.op_line, l.bar_id);
            die("deadlock: no thread can make progress");
        }
    }
    cta() = nullptr; cur() = nullptr;
}

// grid of CTAs, one after the other; launches from several host threads are serialised (the emulator's state is global)
inline std::mutex& launch_mutex() { static std::mutex m; return m; }
inline void launch(unsigned grid, int nthreads, std::function<void()> body)
{
    std::lock_guard<std::mutex> g(launch_mutex());
    for (unsigned b = 0; b < grid; b++) run_cta(nthreads, Idx{b, 0, 0}, Idx{grid, 1, 1}, body);
}

template <class T> inline uint32_t bits(T v) { static_assert(sizeof(T) <= 4, "32-bit payload"); uint32_t u = 0; std::memcpy(&u, &v, sizeof(T)); return u; }
template <class T> inline T unbits(uint32_t u) { T v; std::memcpy(&v, &u, sizeof(T)); return v; }
inline int lane_of() { return cur()->tid & 31; }

// 32-bit payloads directly, 64-bit ones (CUDA allows long long / double) as two shuffles
template <class T> inline T shfl_src(int line, T v, int src)
{
    if constexpr (sizeof(T) <= 4) return unbits<T>(warp_op(OP_SHFL, line, bits(v), src));
    else {
        static_assert(sizeof(T) == 8, "shuffle payload");
        uint64_t u; std::memcpy(&u, &v, 8);
        const uint64_t lo = warp_op(OP_SHFL, line, (uint32_t)u, src), hi = warp_op(OP_SHFL, line, (uint32_t)(u >> 32), src);
        u = lo | (hi << 32); T r; std::memcpy(&r, &u, 8); return r;
    }
}
template <class T> inline T shfl(int line, unsigned, T v, int src) { return shfl_src(line, v, src & 31); }
template <class T> inline T shfl_xor(int line, unsigned, T v, int m) { return shfl_src(line, v, lane_of() ^ m); }
template <class T> inline T shfl_up(int line, unsigned, T v, int d) { const int s = lane_of() - d; return shfl_src(line, v, s < 0 ? lane_of() : s); }
template <class T> inline T shfl_down(int line, unsigned, T v, int d) { const int s = lane_of() + d; return shfl_src(line, v, s > 31 ? lane_of() : s); }

} // namespace simt

#define threadIdx (simt::Idx{(unsigned)simt::cur()->tid, 0, 0})
#define blockIdx (simt::cta()->block)
#define blockDim (simt::cta()->dim)
#define gridDim (simt::cta()->grid)

#define __shfl_sync(...) simt::shfl(__LINE__, __VA_ARGS__)
#define __shfl_xor_sync(...) simt::shfl_xor(__LINE__, __VA_ARGS__)
#define __shfl_up_sync(...) simt::shfl_up(__LINE__, __VA_ARGS__)
#define __shfl_down_sync(...) simt::shfl_down(__LINE__, __VA_ARGS__)
#define __ballot_sync(m, p) simt::warp_op(simt::OP_BALLOT, __LINE__, (p) ? 1u : 0u, 0)
#define __any_sync(m, p) (simt::warp_op(simt::OP_BALLOT, __LINE__, (p) ? 1u : 0u, 0) != 0u)
#define __all_sync(m, p) (simt::warp_op(simt::OP_BALLOT, __LINE__, (p) ? 0u : 1u, 0) == 0u)
#define __syncwarp(...) ((void)simt::warp_op(simt::OP_SYNCWARP, __LINE__, 0u, 0))
#define __reduce_max_sync(m, v) ((int)simt::warp_op(simt::OP_REDUCE_MAX, __LINE__, (uint32_t)(int)(v), 0))
#define __reduce_or_sync(m, v) (simt::warp_op(simt::OP_REDUCE_OR, __LINE__, (uint32_t)(v), 0))
#define __match_any_sync(m, v) (simt::warp_op(simt::OP_MATCH_ANY, __LINE__, (uint32_t)(v), 0))
#define __syncthreads() simt::bar_sync(0, (int)simt::cta()->dim.x)
#define __activemask() 0xFFFFFFFFu
