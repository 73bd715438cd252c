// capi.cu — the C ABI of libb200lz4.so (include/b200lz4.h): device selection, per-thread
// streams and staging, the one-block-per-call entry points the JNI shim binds, and the batch
// entry points (device-resident and host-buffer, the latter as a 3-slot H2D / kernel / D2H
// pipeline).  No codec or hash arithmetic happens on the host: everything is a kernel launch.
#include "../../include/b200lz4.h"
#include "kernels.h"

#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <new>
#include <string>
#include <thread>
#include <vector>
#if defined(__linux__) && !defined(B200_HOST_SIM)
#include <sched.h>
#define B200_HAVE_AFFINITY 1
#endif

namespace b200 {

std::atomic<unsigned long long> g_launch_count{0};
static thread_local char tl_err[256] = "";
static thread_local int tl_status = 0;          // B200LZ4_E_* of the last value-returning call (hashes, digests) on this thread
static thread_local int tl_device = -1;          // -1: not chosen yet (defaults to device 0)

int fail_cuda(cudaError_t e, const char* where)
{
    snprintf(tl_err, sizeof tl_err, "%s: %s", where, cudaGetErrorString(e));
    if (e == cudaErrorNoDevice || e == cudaErrorInsufficientDriver || e == cudaErrorInitializationError)
        return tl_status = B200LZ4_E_NODEVICE;
    return tl_status = B200LZ4_E_CUDA;
}
int fail_arg(const char* what) { snprintf(tl_err, sizeof tl_err, "invalid argument: %s", what); return tl_status = B200LZ4_E_ARG; }

int check_stream_ranges(size_t ns, const uint64_t* src_len, uint64_t src_max, const uint64_t* dst_off, const uint64_t* dst_cap,
                        const void* d_src, const void* d_dst, uint64_t& bytes, uint64_t& room)
{
    bytes = 0; room = 0;
    for (size_t k = 0; k < ns; k++) {
        if (src_len[k] > src_max || dst_cap[k] > (1ull << 47)) return fail_arg("src_len / dst_cap");
        if (dst_off[k] > ~0ull - dst_cap[k]) return fail_arg("a destination range overflows");
        bytes += src_len[k]; room += dst_cap[k];
    }
    if ((bytes && !d_src) || (room && !d_dst)) return fail_arg("null pointer");
    return 0;
}

static int ensure_device()
{
    int cnt = 0;
    cudaError_t e = cudaGetDeviceCount(&cnt);
    if (e != cudaSuccess) return fail_cuda(e, "cudaGetDeviceCount");
    if (cnt <= 0) { snprintf(tl_err, sizeof tl_err, "no CUDA device"); return tl_status = B200LZ4_E_NODEVICE; }
    if (tl_device < 0) {
        // no b200lz4_set_device() on this thread yet: adopt the thread's CURRENT device (0 on a fresh thread) instead of
        // forcing device 0, so a caller that already selected a GPU (torch.cuda.set_device, cudaSetDevice) and hands
        // us device pointers / its stream does not find its current device switched under it
        int cur = 0;
        if (cudaGetDevice(&cur) != cudaSuccess || cur < 0 || cur >= cnt) cur = 0;
        tl_device = cur;
    }
    CK(cudaSetDevice(tl_device));
    return 0;
}

// ---------------------------------------------------------------------------------------------
// Per-block descriptors of one chunk: [total | soff | doff | out] u64, [slen | dcap | res] i32, for nb blocks.
// `out` is what the device hands back per block besides `res`: the packed offsets (compact) or the hashes.
struct Desc {
    uint8_t* base = nullptr; size_t cap = 0;           // allocation, in bytes
    size_t nb = 0;                                     // blocks the layout is cut for
    uint64_t* total() const { return (uint64_t*)base; }
    uint64_t* soff() const { return (uint64_t*)base + 2; }
    uint64_t* doff() const { return soff() + nb; }
    uint64_t* out()  const { return soff() + 2 * nb; }
    int32_t*  slen() const { return (int32_t*)(soff() + 3 * nb); }
    int32_t*  dcap() const { return slen() + nb; }
    int32_t*  res()  const { return slen() + 2 * nb; }
    static size_t bytes(size_t nb) { return 16 + nb * (3 * 8 + 3 * 4); }
    size_t bytes() const { return bytes(nb); }
};

// A pipeline slot: one stream, device staging for a chunk of blocks and its descriptors, pinned and on the device.
struct Slot {
    cudaStream_t st = nullptr;
    cudaEvent_t done = nullptr;
    uint8_t *d_src = nullptr, *d_dst = nullptr; size_t src_cap = 0, dst_cap = 0;
    uint8_t* d_aux = nullptr; size_t aux_cap = 0;      // compacted output (compact_host only)
    uint8_t* h_out = nullptr; size_t h_out_cap = 0;    // pinned bounce for scattered dst slots
    bool scatter = false;                              // retire must copy h_out -> caller slots
    cudaEvent_t drained = nullptr; bool draining = false;
    Desc h, d;                                         // same layout: h is pinned, d its device copy
    size_t i0 = 0, i1 = 0;            // block range in flight
    bool busy = false;
};

static constexpr int    NSLOTS = 3;
static size_t chunk_span_init() { const char* e = getenv("B200LZ4_CHUNK_MB"); size_t mb = e ? (size_t)atol(e) : 256; if (mb < 1) mb = 1; return mb << 20; }
const size_t CHUNK_SPAN = chunk_span_init();           // bytes of src (and of dst) per pipeline chunk: >= 4096 64-KiB blocks,
                                                           // i.e. at least two full waves of warps on 132 SMs per launch

struct Ctx {
    int device = -1;
    Slot slot[NSLOTS];
    // one-block path
    uint8_t* h_bounce = nullptr; size_t bounce_cap = 0;    // pinned: [src | dst]
    FrameScratch frame;                                    // the frame writer (containers.cu)
    FrameReadScratch frame_read;                           // the frame reader (frame.cu)
    SideStream side;                                       // both frame calls' checksum stream
    ~Ctx() { /* process teardown frees device memory; explicit frees would race CUDA shutdown */ }
};

// Contexts (streams + staging) are owned by one thread at a time.  A thread keeps one per device it has used; when
// the thread exits they go to a process-wide idle pool and the next new thread on that device picks them up, so a
// server that churns threads (or a thread that alternates devices) does not grow device memory without bound.  No CUDA
// call happens at thread exit (nothing here can race the runtime's own teardown); the pool itself is never destroyed.
static std::atomic<int> g_contexts{0};
struct CtxPool { std::mutex mu; std::vector<Ctx*> idle; };
static CtxPool& ctx_pool() { static CtxPool* p = new CtxPool(); return *p; }
struct ThreadCtxs {
    std::vector<Ctx*> mine;
    ~ThreadCtxs()
    {
        if (mine.empty()) return;
        CtxPool& p = ctx_pool();
        std::lock_guard<std::mutex> g(p.mu);
        for (Ctx* c : mine) p.idle.push_back(c);
    }
};
static thread_local ThreadCtxs tl_ctxs;
static thread_local Ctx* tl_ctx = nullptr;          // the context of tl_device (cache of the lookup below)

static int get_ctx(Ctx** out)
{
    int rc = ensure_device();
    if (rc) return rc;
    if (tl_ctx && tl_ctx->device != tl_device) tl_ctx = nullptr;        // device switched on this thread
    if (!tl_ctx) {
        for (Ctx* c : tl_ctxs.mine) if (c->device == tl_device) { tl_ctx = c; break; }
    }
    if (!tl_ctx) {
        CtxPool& p = ctx_pool();
        std::lock_guard<std::mutex> g(p.mu);
        for (size_t k = 0; k < p.idle.size(); k++)
            if (p.idle[k]->device == tl_device) { tl_ctx = p.idle[k]; p.idle.erase(p.idle.begin() + (long)k); break; }
        if (tl_ctx) tl_ctxs.mine.push_back(tl_ctx);
    }
    if (!tl_ctx) {
        Ctx* c = new (std::nothrow) Ctx();
        if (!c) return fail_arg("out of host memory");
        c->device = tl_device;
        for (int s = 0; s < NSLOTS; s++) {
            cudaError_t e = cudaStreamCreateWithFlags(&c->slot[s].st, cudaStreamNonBlocking);
            if (e == cudaSuccess) e = cudaEventCreateWithFlags(&c->slot[s].done, cudaEventDisableTiming);
            if (e == cudaSuccess) e = cudaEventCreateWithFlags(&c->slot[s].drained, cudaEventDisableTiming);
            if (e != cudaSuccess) {
                for (int t = 0; t <= s; t++) {
                    if (c->slot[t].st) cudaStreamDestroy(c->slot[t].st);
                    if (c->slot[t].done) cudaEventDestroy(c->slot[t].done);
                    if (c->slot[t].drained) cudaEventDestroy(c->slot[t].drained);
                }
                delete c;
                return fail_cuda(e, "creating the pipeline streams");
            }
        }
        tl_ctxs.mine.push_back(c);
        tl_ctx = c;
        g_contexts.fetch_add(1, std::memory_order_relaxed);
    }
    *out = tl_ctx;
    return 0;
}

// A pipeline call that fails half way (a CUDA error, or an argument error found at a later chunk) must not leave
// chunks in flight: the next call on this thread would retire them into ITS result array with the old block indices.
// The guard waits for whatever was queued and clears the slots' bookkeeping unless the call ran to completion.
static void ctx_abandon(Ctx* c)
{
    for (int k = 0; k < NSLOTS; k++) {
        Slot& s = c->slot[k];
        if (s.busy || s.draining) cudaStreamSynchronize(s.st);       // result of the wait is irrelevant here
        s.busy = false; s.draining = false; s.scatter = false;
    }
}
struct PipelineGuard {
    Ctx* c; bool completed = false;
    explicit PipelineGuard(Ctx* c_) : c(c_) {}
    ~PipelineGuard() { if (!completed) ctx_abandon(c); }
};

// the thread's context, with its side stream when `side` asks for it
static int get_frame_ctx(Ctx** c, SideStream** side)
{
    int rc = get_ctx(c); if (rc) return rc;
    if (!side) return 0;
    SideStream& s = (*c)->side;
    if (!s.st) {
        cudaError_t e = cudaStreamCreateWithFlags(&s.st, cudaStreamNonBlocking);
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&s.fork, cudaEventDisableTiming);
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&s.join, cudaEventDisableTiming);
        if (e != cudaSuccess) {
            if (s.st) cudaStreamDestroy(s.st);
            if (s.fork) cudaEventDestroy(s.fork);
            s = SideStream{};
            return fail_cuda(e, "creating the frame calls' checksum stream");
        }
    }
    *side = &s;
    return 0;
}

int get_frame_scratch(FrameScratch** out, SideStream** side, cudaStream_t* idle)
{
    Ctx* c; int rc = get_frame_ctx(&c, side); if (rc) return rc;
    *out = &c->frame;
    if (idle) *idle = c->slot[0].st;           // a pipeline call leaves its slots drained (run_pipeline, ctx_abandon)
    return 0;
}

int get_frame_read_scratch(FrameReadScratch** out, SideStream** side, cudaStream_t* idle)
{
    Ctx* c; int rc = get_frame_ctx(&c, side); if (rc) return rc;
    *out = &c->frame_read;
    if (idle) *idle = c->slot[0].st;           // a pipeline call leaves its slots drained (run_pipeline, ctx_abandon)
    return 0;
}

// Grow-or-keep staging: a buffer smaller than `need` bytes is replaced by one with need >> slack_shift more room plus
// 4 KiB, so calls of about the same size keep their buffers.  Whatever still reads or writes the old buffer must be done.
int reserve_device(uint8_t*& p, size_t& cap, size_t need, int slack_shift)
{
    if (need <= cap) return 0;
    if (p) CK(cudaFree(p));
    p = nullptr; cap = 0;
    const size_t c = need + (need >> slack_shift) + 4096;
    CK(cudaMalloc(&p, c)); cap = c;
    return 0;
}
int reserve_pinned(uint8_t*& p, size_t& cap, size_t need)
{
    if (need <= cap) return 0;
    if (p) CK(cudaFreeHost(p));
    p = nullptr; cap = 0;
    const size_t c = need + (need >> 2) + 4096;
    CK(cudaHostAlloc(&p, c, cudaHostAllocDefault)); cap = c;
    return 0;
}

static int slot_reserve(Slot& s, size_t src_bytes, size_t dst_bytes, size_t nblocks, size_t aux_bytes = 0)
{
    if (s.draining) { CK(cudaEventSynchronize(s.drained)); s.draining = false; }
    int rc = reserve_device(s.d_aux, s.aux_cap, aux_bytes);
    if (!rc) rc = reserve_device(s.d_src, s.src_cap, src_bytes);
    if (!rc) rc = reserve_device(s.d_dst, s.dst_cap, dst_bytes);
    if (rc || nblocks <= s.h.nb) return rc;
    size_t nb = nblocks + (nblocks >> 1) + 64;
    nb = (nb + 1) & ~size_t(1);                        // keeps the i32 arrays 8-byte aligned
    s.h.nb = s.d.nb = 0;                               // a failed reserve below frees the old buffer: the next call must allocate
    rc = reserve_device(s.d.base, s.d.cap, Desc::bytes(nb));
    if (!rc) rc = reserve_pinned(s.h.base, s.h.cap, Desc::bytes(nb));
    if (!rc) s.h.nb = s.d.nb = nb;
    return rc;
}

enum Op { OP_COMPRESS_FAST, OP_COMPRESS_HC, OP_DEC_SAFE, OP_DEC_FAST };

static cudaError_t launch_op(Op op, const BatchArgs& a, int param, cudaStream_t st)
{
    g_launch_count.fetch_add(1, std::memory_order_relaxed);
    switch (op) {
    case OP_COMPRESS_FAST: return launch_compress_fast(a, param, st);
    case OP_COMPRESS_HC:   return launch_compress_hc(a, param, st);
    case OP_DEC_SAFE:      return launch_decompress_safe(a, st);
    default:               return launch_decompress_fast(a, st);
    }
}

// One chunk of a host-buffer call: blocks [i0, i0 + nb), their source bytes [s_lo, s_lo + s_span) and, when the call
// has dst slots, their dst bytes [d_lo, d_lo + d_span).
struct Chunk { size_t i0, nb; uint64_t s_lo, d_lo; size_t s_span, d_span; };

// The host-buffer pipeline every host-buffer call runs.  It cuts blocks [0, n) into chunks of at most CHUNK_BLOCKS blocks
// and CHUNK_SPAN bytes of source (and of dst, when dst_off is given) and runs them round-robin over the NSLOTS streams:
//   stage(Slot&, const Chunk&)  reserves the slot's buffers and queues the chunk's copies in, its launches and its copies
//                               back on s.st; the driver then records s.done;
//   retire(Slot&)               hands the chunk [s.i0, s.i1) back to the caller, after s.done.
// A slot's chunk is retired before the slot takes the next one and the last ones in block order, so results come back in
// block order; the call returns after every `drained` event a retire recorded.  Blocks must ascend in src (and in dst,
// without overlapping there); order_msg is the error otherwise.
template <class Stage, class Retire>
static int run_pipeline(size_t n, const uint64_t* src_off, const int32_t* src_len, const uint64_t* dst_off,
                        const int32_t* dst_cap, const char* order_msg, Stage stage, Retire retire)
{
    Ctx* c; int rc = get_ctx(&c); if (rc) return rc;
    PipelineGuard guard(c);
    auto finish = [&](Slot& s) -> int {
        if (!s.busy) return 0;
        CK(cudaEventSynchronize(s.done));
        const int r = retire(s); if (r) return r;
        s.busy = false;
        return 0;
    };
    size_t i0 = 0; int cur = 0;
    while (i0 < n) {
        // ---- pick the chunk [i0, i1).  Negative sizes span no bytes: they are per-block errors in the reference
        // (lz4.c:1324, 1953), and the kernels report them.
        const uint64_t s_lo = src_off[i0], d_lo = dst_off ? dst_off[i0] : 0;
        uint64_t s_hi = s_lo, d_hi = d_lo;
        size_t i1 = i0;
        while (i1 < n && i1 - i0 < CHUNK_BLOCKS) {
            if (src_off[i1] < s_lo || (dst_off && (dst_off[i1] < d_lo || (i1 > i0 && dst_off[i1] < d_hi)))) return fail_arg(order_msg);
            const uint64_t se = src_off[i1] + (uint64_t)(src_len[i1] > 0 ? src_len[i1] : 0);
            const uint64_t de = dst_off ? dst_off[i1] + (uint64_t)(dst_cap[i1] > 0 ? dst_cap[i1] : 0) : 0;
            const uint64_t ns = se > s_hi ? se : s_hi, nd = de > d_hi ? de : d_hi;
            if (i1 > i0 && (ns - s_lo > CHUNK_SPAN || nd - d_lo > CHUNK_SPAN)) break;
            s_hi = ns; d_hi = nd; i1++;
        }
        Slot& s = c->slot[cur];
        rc = finish(s); if (rc) return rc;
        rc = stage(s, Chunk{ i0, i1 - i0, s_lo, d_lo, (size_t)(s_hi - s_lo), (size_t)(d_hi - d_lo) }); if (rc) return rc;
        CK(cudaEventRecord(s.done, s.st));
        s.busy = true; s.i0 = i0; s.i1 = i1;
        i0 = i1; cur = (cur + 1) % NSLOTS;
    }
    for (int k = 0; k < NSLOTS; k++) { rc = finish(c->slot[(cur + k) % NSLOTS]); if (rc) return rc; }
    for (Slot& s : c->slot) if (s.draining) { CK(cudaEventSynchronize(s.drained)); s.draining = false; }
    guard.completed = true;
    return 0;
}

// Host-buffer batch: chunk, stage, launch, copy back.  Blocks ascend in src and dst.
static int host_batch(Op op, const uint8_t* src_base, const uint64_t* src_off, const int32_t* src_len,
                      uint8_t* dst_base, const uint64_t* dst_off, const int32_t* dst_cap,
                      int32_t* result, size_t n, int param)
{
    if (n == 0) return 0;
    if (!src_base || !src_off || !src_len || !dst_base || !dst_off || !dst_cap || !result) return fail_arg("null pointer");
    auto stage = [&](Slot& s, const Chunk& ch) -> int {
        int rc = slot_reserve(s, ch.s_span + 16, ch.d_span + 16, ch.nb); if (rc) return rc;
        // keep the source's 16-byte phase so aligned inputs stay aligned on the device
        const size_t s_phase = (size_t)((uintptr_t)(src_base + ch.s_lo) & 15), d_phase = (size_t)((uintptr_t)(dst_base + ch.d_lo) & 15);
        for (size_t k = 0; k < ch.nb; k++) {
            s.h.soff()[k] = src_off[ch.i0 + k] - ch.s_lo + s_phase;
            s.h.doff()[k] = dst_off[ch.i0 + k] - ch.d_lo + d_phase;
            s.h.slen()[k] = src_len[ch.i0 + k];
            s.h.dcap()[k] = dst_cap[ch.i0 + k];
        }
        CK(cudaMemcpyAsync(s.d.base, s.h.base, s.h.bytes(), cudaMemcpyHostToDevice, s.st));
        if (ch.s_span) CK(cudaMemcpyAsync(s.d_src + s_phase, src_base + ch.s_lo, ch.s_span, cudaMemcpyHostToDevice, s.st));
        BatchArgs a{ s.d_src, s.d.soff(), s.d.slen(), s.d_dst, s.d.doff(), s.d.dcap(), s.d.res(), ch.nb };
        CK(launch_op(op, a, param, s.st));
        CK(cudaMemcpyAsync(s.h.res(), s.d.res(), ch.nb * sizeof(int32_t), cudaMemcpyDeviceToHost, s.st));
        if (!ch.d_span) return 0;
        if (n == 1) {
            // one block per call (the JNI shim's shape): the caller's bytes behind the result stay untouched, like in the
            // reference (a decoder called with maxDestLen = "rest of my buffer" must not clobber what lies further along),
            // and no stale staging bytes of another call leave the device.  Costs one more round trip of a few bytes.
            CK(cudaStreamSynchronize(s.st));
            const int32_t r = s.h.res()[0];
            const size_t produced = op == OP_DEC_FAST ? (r >= 0 ? ch.d_span : 0) : (size_t)(r > 0 ? r : 0);
            if (produced) CK(cudaMemcpyAsync(dst_base + ch.d_lo, s.d_dst + d_phase, produced < ch.d_span ? produced : ch.d_span, cudaMemcpyDeviceToHost, s.st));
            return 0;
        }
        // copy back: when the dst slots are back to back (the normal layout) one DMA lands straight in
        // the caller's memory; otherwise the span goes to a pinned bounce buffer and retire scatters
        // the slots, so caller bytes BETWEEN non-adjacent slots are never touched
        bool contiguous = true;
        uint64_t end = ch.d_lo;
        for (size_t k = ch.i0; k < ch.i0 + ch.nb && contiguous; k++) {
            if (dst_off[k] != end) contiguous = false;
            end = dst_off[k] + (uint64_t)(dst_cap[k] > 0 ? dst_cap[k] : 0);
        }
        if (contiguous) {
            CK(cudaMemcpyAsync(dst_base + ch.d_lo, s.d_dst + d_phase, ch.d_span, cudaMemcpyDeviceToHost, s.st));
        } else {
            rc = reserve_pinned(s.h_out, s.h_out_cap, ch.d_span); if (rc) return rc;
            CK(cudaMemcpyAsync(s.h_out, s.d_dst + d_phase, ch.d_span, cudaMemcpyDeviceToHost, s.st));
            s.scatter = true;
        }
        return 0;
    };
    auto retire = [&](Slot& s) -> int {
        memcpy(result + s.i0, s.h.res(), (s.i1 - s.i0) * sizeof(int32_t));
        if (s.scatter) {
            const uint64_t d_lo = dst_off[s.i0];
            for (size_t k = s.i0; k < s.i1; k++)
                if (dst_cap[k] > 0) memcpy(dst_base + dst_off[k], s.h_out + (dst_off[k] - d_lo), (size_t)dst_cap[k]);
            s.scatter = false;
        }
        return 0;
    };
    return run_pipeline(n, src_off, src_len, dst_off, dst_cap, "blocks must ascend and not overlap in dst", stage, retire);
}

template <typename W>
static int hash_host_batch(int bits, const uint8_t* base, const uint64_t* off, const int32_t* len, uint64_t seed,
                           W* out, size_t n)
{
    if (n == 0) return 0;
    if (!base || !off || !len || !out) return fail_arg("null pointer");
    auto stage = [&](Slot& s, const Chunk& ch) -> int {
        int rc = slot_reserve(s, ch.s_span + 16, 16, ch.nb); if (rc) return rc;
        const size_t phase = (size_t)((uintptr_t)(base + ch.s_lo) & 15);
        for (size_t k = 0; k < ch.nb; k++) { s.h.soff()[k] = off[ch.i0 + k] - ch.s_lo + phase; s.h.slen()[k] = len[ch.i0 + k]; }
        CK(cudaMemcpyAsync(s.d.base, s.h.base, s.h.bytes(), cudaMemcpyHostToDevice, s.st));
        if (ch.s_span) CK(cudaMemcpyAsync(s.d_src + phase, base + ch.s_lo, ch.s_span, cudaMemcpyHostToDevice, s.st));
        g_launch_count.fetch_add(1, std::memory_order_relaxed);
        const bool few_long = ch.s_span / ch.nb >= XXH_LONG_AVG;
        if (bits == 32) CK((few_long ? launch_xxh32_long : launch_xxh32)(
                               s.d_src, s.d.soff(), s.d.slen(), (uint32_t)seed, (uint32_t*)s.d.out(), ch.nb, s.st));
        else            CK((few_long ? launch_xxh64_long : launch_xxh64)(
                               s.d_src, s.d.soff(), s.d.slen(), seed, s.d.out(), ch.nb, s.st));
        CK(cudaMemcpyAsync(s.h.out(), s.d.out(), ch.nb * sizeof(W), cudaMemcpyDeviceToHost, s.st));
        return 0;
    };
    auto retire = [&](Slot& s) -> int { memcpy(out + s.i0, s.h.out(), (s.i1 - s.i0) * sizeof(W)); return 0; };
    return run_pipeline(n, off, len, nullptr, nullptr, "buffers must ascend", stage, retire);
}

// one block, host buffers: the n = 1 case of the host batch path
static int one_block(Op op, const char* src, int src_len, char* dst, int dst_cap, int param)
{
    const uint64_t zero = 0;
    int32_t res = 0;
    static const char dummy = 0;
    if (!src) src = &dummy;
    char local_dst = 0;
    if (!dst) { dst = &local_dst; if (dst_cap > 0) return fail_arg("dst is NULL"); }
    int rc = host_batch(op, (const uint8_t*)src, &zero, &src_len, (uint8_t*)dst, &zero, &dst_cap, &res, 1, param);
    if (rc) return rc;
    return res;
}

// Pin the calling WORKER thread to the CPUs of the NUMA node its GPU hangs off (sysfs: the PCI device's numa_node and the
// node's cpulist).  Staging and descriptor buffers a worker allocates then land on that node (first touch), and its DMA
// descriptors are written by a core next to the root complex.  Round 1's 8-GPU end-to-end run scaled 0.355 with every
// thread floating over both sockets.  Best effort: any failure leaves the thread where it was.
static void bind_worker_to_device_node(int device)
{
#ifdef B200_HAVE_AFFINITY
    char bus[32] = "";
    if (cudaDeviceGetPCIBusId(bus, sizeof bus, device) != cudaSuccess) return;
    for (char* q = bus; *q; q++) if (*q >= 'A' && *q <= 'Z') *q = char(*q - 'A' + 'a');
    char path[160];
    snprintf(path, sizeof path, "/sys/bus/pci/devices/%s/numa_node", bus);
    FILE* f = fopen(path, "r"); if (!f) return;
    int node = -1; const int got = fscanf(f, "%d", &node); fclose(f);
    if (got != 1 || node < 0) return;
    snprintf(path, sizeof path, "/sys/devices/system/node/node%d/cpulist", node);
    f = fopen(path, "r"); if (!f) return;
    char list[1024] = ""; const bool ok = fgets(list, sizeof list, f) != nullptr; fclose(f);
    if (!ok) return;
    cpu_set_t want; CPU_ZERO(&want);
    for (char* q = list; *q; ) {                                   // "0-31,64-95"
        char* e; const long a = strtol(q, &e, 10); if (e == q) break;
        long b = a; q = e;
        if (*q == '-') { b = strtol(q + 1, &e, 10); q = e; }
        for (long c = a; c <= b && c < CPU_SETSIZE; c++) CPU_SET((int)c, &want);
        if (*q == ',') q++; else break;
    }
    cpu_set_t cur;
    if (sched_getaffinity(0, sizeof cur, &cur) != 0) return;
    cpu_set_t both; CPU_AND(&both, &cur, &want);                   // never widen what the process was given (cgroups, taskset)
    if (CPU_COUNT(&both) > 0) sched_setaffinity(0, sizeof both, &both);
#else
    (void)device;
#endif
}

// ---- one process, several GPUs: contiguous block ranges, one worker thread (own device, own context) per GPU
template <class ShardFn>
static int run_sharded(size_t n, const int* devices, int ndev, ShardFn shard)
{
    if (ndev < 1 || ndev > 64) return fail_arg("ndev must be 1..64");
    int cnt = b200lz4_device_count();
    if (cnt < 0) return cnt;
    for (int g = 0; g < ndev; g++) {
        const int d = devices ? devices[g] : g;
        if (d < 0 || d >= cnt) return fail_arg("device index in devices[]");
    }
    std::vector<int> rc((size_t)ndev, 0);
    std::vector<std::string> msg((size_t)ndev);
    std::vector<std::thread> th;
    auto body = [&](int g) {
        const size_t lo = n * (size_t)g / (size_t)ndev, hi = n * (size_t)(g + 1) / (size_t)ndev;
        if (hi == lo) return;
        int r = b200lz4_set_device(devices ? devices[g] : g);       // thread-local: this worker's device
        if (r == 0 && g > 0) bind_worker_to_device_node(devices ? devices[g] : g);      // (shard 0 runs on the caller's thread: its affinity is the caller's business)
        if (r == 0) r = shard(lo, hi - lo);
        rc[(size_t)g] = r;
        if (r) msg[(size_t)g] = tl_err;
    };
    try {
        for (int g = 1; g < ndev; g++) th.emplace_back(body, g);
    } catch (...) {
        for (auto& t : th) t.join();
        return fail_arg("cannot start a worker thread");
    }
    const int my_device = tl_device;
    int my_cuda_device = -1;
    if (cudaGetDevice(&my_cuda_device) != cudaSuccess) my_cuda_device = -1;
    body(0);                                                        // shard 0 runs on the calling thread
    for (auto& t : th) t.join();
    tl_device = my_device;                                          // the caller keeps its device, in the library and in CUDA
    if (my_cuda_device >= 0) cudaSetDevice(my_cuda_device);
    for (int g = 0; g < ndev; g++)
        if (rc[(size_t)g]) {
            snprintf(tl_err, sizeof tl_err, "device %d: %s", devices ? devices[g] : g, msg[(size_t)g].c_str());
            return tl_status = rc[(size_t)g];
        }
    return 0;
}

static int multi_host_batch(Op op, const uint8_t* src_base, const uint64_t* src_off, const int32_t* src_len,
                            uint8_t* dst_base, const uint64_t* dst_off, const int32_t* dst_cap,
                            int32_t* result, size_t n, int param, const int* devices, int ndev)
{
    if (n == 0) return 0;
    if (!src_base || !src_off || !src_len || !dst_base || !dst_off || !dst_cap || !result) return fail_arg("null pointer");
    return run_sharded(n, devices, ndev, [&](size_t lo, size_t cnt) {
        return host_batch(op, src_base, src_off + lo, src_len + lo, dst_base, dst_off + lo, dst_cap + lo, result + lo, cnt, param);
    });
}

} // namespace b200

using namespace b200;

extern "C" {

int b200lz4_version(void) { return B200LZ4_VERSION; }

int b200lz4_device_count(void)
{
    int cnt = 0;
    cudaError_t e = cudaGetDeviceCount(&cnt);
    if (e != cudaSuccess) return fail_cuda(e, "cudaGetDeviceCount");
    return cnt;
}

int b200lz4_set_device(int device)
{
    int cnt = b200lz4_device_count();
    if (cnt < 0) return cnt;
    if (device < 0 || device >= cnt) return fail_arg("device index");
    tl_device = device;
    CK(cudaSetDevice(device));
    return 0;
}

const char* b200lz4_last_error(void) { return tl_err; }
int b200lz4_last_status(void) { return tl_status; }

int b200lz4_host_register(void* p, size_t bytes)
{
    int rc = ensure_device(); if (rc) return rc;
    CK(cudaHostRegister(p, bytes, cudaHostRegisterPortable));
    return 0;
}
int b200lz4_host_unregister(void* p)
{
    int rc = ensure_device(); if (rc) return rc;
    CK(cudaHostUnregister(p));
    return 0;
}

int b200lz4_compressBound(int n)
{   // pure size arithmetic (lz4.h:212); LZ4Utils.maxCompressedLength must equal it (LZ4Test.java:80-87)
    return ((unsigned)n > 0x7E000000u) ? 0 : n + n / 255 + 16;
}

int b200lz4_compress_default(const char* src, char* dst, int srcSize, int dstCapacity)
{
    if (srcSize < 0 || (unsigned)srcSize > 0x7E000000u || dstCapacity < 0) return 0;  // lz4.c:1324; no room at all
    return one_block(OP_COMPRESS_FAST, src, srcSize, dst, dstCapacity, srcSize <= 65536 ? 65536 : 0);
}
int b200lz4_compress_HC(const char* src, char* dst, int srcSize, int dstCapacity, int level)
{
    if (srcSize < 0 || (unsigned)srcSize > 0x7E000000u || dstCapacity < 0) return 0;
    return one_block(OP_COMPRESS_HC, src, srcSize, dst, dstCapacity, level);
}
int b200lz4_decompress_safe(const char* src, char* dst, int compressedSize, int dstCapacity)
{
    if (!src || dstCapacity < 0) return -1;                                           // lz4.c:1953
    if (compressedSize < 0) return -1;
    return one_block(OP_DEC_SAFE, src, compressedSize, dst, dstCapacity, 0);
}
int b200lz4_decompress_fast_bounded(const char* src, int srcAvail, char* dst, int originalSize)
{
    if (!src || originalSize < 0 || srcAvail < 0) return -1;
    return one_block(OP_DEC_FAST, src, srcAvail, dst, originalSize, 0);
}

uint32_t b200xxh32(const void* input, size_t len, uint32_t seed)
{
    const uint64_t zero = 0; int32_t l = (int32_t)len; uint32_t out = 0; static const char dummy = 0;
    tl_status = 0;
    if (len > 0x7FFFFFFFu) { fail_arg("len > 2^31-1"); return 0; }
    if (hash_host_batch<uint32_t>(32, (const uint8_t*)(input ? input : &dummy), &zero, &l, seed, &out, 1)) return 0;
    return out;
}
uint64_t b200xxh64(const void* input, size_t len, uint64_t seed)
{
    const uint64_t zero = 0; int32_t l = (int32_t)len; uint64_t out = 0; static const char dummy = 0;
    tl_status = 0;
    if (len > 0x7FFFFFFFu) { fail_arg("len > 2^31-1"); return 0; }
    if (hash_host_batch<uint64_t>(64, (const uint8_t*)(input ? input : &dummy), &zero, &l, seed, &out, 1)) return 0;
    return out;
}

// ---- streaming state: device-resident struct + a pinned staging area, one stream per handle
struct StreamHandle {
    int bits; int device; void* d_state; uint8_t* d_buf; size_t buf_cap; cudaStream_t st; void* h_out;
};
static void* stream_create(int bits, uint64_t seed)
{
    if (ensure_device()) return nullptr;
    StreamHandle* h = new (std::nothrow) StreamHandle();
    if (!h) return nullptr;
    h->bits = bits; h->device = tl_device; h->d_buf = nullptr; h->buf_cap = 0;
    if (cudaStreamCreateWithFlags(&h->st, cudaStreamNonBlocking) != cudaSuccess ||
        cudaMalloc(&h->d_state, bits == 32 ? sizeof(Xxh32State) : sizeof(Xxh64State)) != cudaSuccess ||
        cudaHostAlloc(&h->h_out, 8, cudaHostAllocDefault) != cudaSuccess) { fail_cuda(cudaGetLastError(), "stream_create"); delete h; return nullptr; }
    g_launch_count.fetch_add(1, std::memory_order_relaxed);
    if (bits == 32) launch_xxh32_stream((Xxh32State*)h->d_state, XXH_OP_RESET, (uint32_t)seed, nullptr, 0, h->st);
    else            launch_xxh64_stream((Xxh64State*)h->d_state, XXH_OP_RESET, seed, nullptr, 0, h->st);
    return h;
}
static void stream_reset(void* hv, uint64_t seed)
{
    StreamHandle* h = (StreamHandle*)hv; if (!h) return;
    cudaSetDevice(h->device);
    g_launch_count.fetch_add(1, std::memory_order_relaxed);
    if (h->bits == 32) launch_xxh32_stream((Xxh32State*)h->d_state, XXH_OP_RESET, (uint32_t)seed, nullptr, 0, h->st);
    else               launch_xxh64_stream((Xxh64State*)h->d_state, XXH_OP_RESET, seed, nullptr, 0, h->st);
}
static int stream_update(void* hv, const void* input, size_t len)
{
    StreamHandle* h = (StreamHandle*)hv; if (!h) return fail_arg("null state");
    if (len == 0) return 0;
    CK(cudaSetDevice(h->device));
    if (len > h->buf_cap) CK(cudaStreamSynchronize(h->st));
    const int rc = reserve_device(h->d_buf, h->buf_cap, len, 1); if (rc) return rc;       // half again: update sizes often keep rising
    CK(cudaMemcpyAsync(h->d_buf, input, len, cudaMemcpyHostToDevice, h->st));
    g_launch_count.fetch_add(1, std::memory_order_relaxed);
    if (h->bits == 32) CK(launch_xxh32_stream((Xxh32State*)h->d_state, XXH_OP_UPDATE, 0, h->d_buf, len, h->st));
    else               CK(launch_xxh64_stream((Xxh64State*)h->d_state, XXH_OP_UPDATE, 0, h->d_buf, len, h->st));
    CK(cudaStreamSynchronize(h->st));          // the caller may reuse `input` as soon as we return
    return 0;
}
static uint64_t stream_digest(void* hv)
{
    tl_status = 0;
    StreamHandle* h = (StreamHandle*)hv; if (!h) { fail_arg("null state"); return 0; }
    cudaSetDevice(h->device);
    g_launch_count.fetch_add(1, std::memory_order_relaxed);
    if (h->bits == 32) {
        launch_xxh32_stream((Xxh32State*)h->d_state, XXH_OP_DIGEST, 0, nullptr, 0, h->st);
        cudaMemcpyAsync(h->h_out, &((Xxh32State*)h->d_state)->digest, 4, cudaMemcpyDeviceToHost, h->st);
    } else {
        launch_xxh64_stream((Xxh64State*)h->d_state, XXH_OP_DIGEST, 0, nullptr, 0, h->st);
        cudaMemcpyAsync(h->h_out, &((Xxh64State*)h->d_state)->digest, 8, cudaMemcpyDeviceToHost, h->st);
    }
    cudaError_t e = cudaStreamSynchronize(h->st);
    if (e != cudaSuccess) { fail_cuda(e, "stream_digest"); return 0; }
    return h->bits == 32 ? (uint64_t)*(uint32_t*)h->h_out : *(uint64_t*)h->h_out;
}
static void stream_free(void* hv)
{
    StreamHandle* h = (StreamHandle*)hv; if (!h) return;
    cudaSetDevice(h->device);
    cudaStreamSynchronize(h->st);
    cudaFree(h->d_state); if (h->d_buf) cudaFree(h->d_buf); cudaFreeHost(h->h_out); cudaStreamDestroy(h->st);
    delete h;
}

void*    b200xxh32_create(uint32_t seed) { return stream_create(32, seed); }
void     b200xxh32_reset(void* s, uint32_t seed) { stream_reset(s, seed); }
int      b200xxh32_update(void* s, const void* in, size_t len) { return stream_update(s, in, len); }
uint32_t b200xxh32_digest(void* s) { return (uint32_t)stream_digest(s); }
void     b200xxh32_free(void* s) { stream_free(s); }
void*    b200xxh64_create(uint64_t seed) { return stream_create(64, seed); }
void     b200xxh64_reset(void* s, uint64_t seed) { stream_reset(s, seed); }
int      b200xxh64_update(void* s, const void* in, size_t len) { return stream_update(s, in, len); }
uint64_t b200xxh64_digest(void* s) { return stream_digest(s); }
void     b200xxh64_free(void* s) { stream_free(s); }

// ---- device-resident batches
#define DEV_BATCH(OP, PARAM) \
    int rc = ensure_device(); if (rc) return rc; \
    if (n > 0xFFFFFFFFull) return fail_arg("n"); \
    BatchArgs a{ src_base, src_off, src_len, dst_base, dst_off, dst_cap, result, n }; \
    CK(launch_op(OP, a, PARAM, (cudaStream_t)stream)); \
    return 0;

int b200lz4_compress_fast_batch_dev(const uint8_t* src_base, const uint64_t* src_off, const int32_t* src_len,
                                    uint8_t* dst_base, const uint64_t* dst_off, const int32_t* dst_cap,
                                    int32_t* result, size_t n, int max_src_len, void* stream)
{ DEV_BATCH(OP_COMPRESS_FAST, max_src_len) }
int b200lz4_compress_hc_batch_dev(const uint8_t* src_base, const uint64_t* src_off, const int32_t* src_len,
                                  uint8_t* dst_base, const uint64_t* dst_off, const int32_t* dst_cap,
                                  int32_t* result, size_t n, int level, void* stream)
{ DEV_BATCH(OP_COMPRESS_HC, level) }
int b200lz4_decompress_safe_batch_dev(const uint8_t* src_base, const uint64_t* src_off, const int32_t* src_len,
                                      uint8_t* dst_base, const uint64_t* dst_off, const int32_t* dst_cap,
                                      int32_t* result, size_t n, void* stream)
{ DEV_BATCH(OP_DEC_SAFE, 0) }
int b200lz4_decompress_fast_batch_dev(const uint8_t* src_base, const uint64_t* src_off, const int32_t* src_len,
                                      uint8_t* dst_base, const uint64_t* dst_off, const int32_t* dst_cap,
                                      int32_t* result, size_t n, void* stream)
{ DEV_BATCH(OP_DEC_FAST, 0) }

int b200xxh32_batch_dev(const uint8_t* base, const uint64_t* off, const int32_t* len, uint32_t seed, uint32_t* out, size_t n, void* stream)
{
    int rc = ensure_device(); if (rc) return rc;
    g_launch_count.fetch_add(1, std::memory_order_relaxed);
    CK(launch_xxh32(base, off, len, seed, out, n, (cudaStream_t)stream));
    return 0;
}
int b200xxh64_batch_dev(const uint8_t* base, const uint64_t* off, const int32_t* len, uint64_t seed, uint64_t* out, size_t n, void* stream)
{
    int rc = ensure_device(); if (rc) return rc;
    g_launch_count.fetch_add(1, std::memory_order_relaxed);
    CK(launch_xxh64(base, off, len, seed, out, n, (cudaStream_t)stream));
    return 0;
}

// ---- device-resident packing and the cross-GPU stitch (SURVEY.md 8e "optional next", (f)-4)
int b200lz4_compact_dev(const uint8_t* slots, const uint64_t* slot_off, const int32_t* lens, uint8_t* out, uint64_t* out_off,
                        uint64_t* total, size_t n, void* stream)
{
    int rc = ensure_device(); if (rc) return rc;
    if (n > 0xFFFFFFFFull) return fail_arg("n");
    if (!total || (n && (!slots || !slot_off || !lens || !out || !out_off))) return fail_arg("null pointer");
    if (n == 0) { CK(cudaMemsetAsync(total, 0, sizeof(uint64_t), (cudaStream_t)stream)); return 0; }
    g_launch_count.fetch_add(2, std::memory_order_relaxed);
    CK(launch_compact(slots, slot_off, lens, out, out_off, total, n, (cudaStream_t)stream));
    return 0;
}

int b200lz4_stitch_shards_dev(const void* const* shard_ptr, const int* shard_dev, const uint64_t* shard_total, int nshard,
                              void* dst, int dst_dev, size_t dst_capacity, uint64_t* shard_pos)
{
    if (nshard < 1 || nshard > 64) return fail_arg("nshard must be 1..64");
    if (!shard_ptr || !shard_dev || !shard_total || !dst) return fail_arg("null pointer");
    int cnt = b200lz4_device_count();
    if (cnt < 0) return cnt;
    if (dst_dev < 0 || dst_dev >= cnt) return fail_arg("dst_dev");
    uint64_t acc = 0;
    std::vector<uint64_t> pos((size_t)nshard);
    for (int g = 0; g < nshard; g++) {
        if (shard_dev[g] < 0 || shard_dev[g] >= cnt) return fail_arg("device index in shard_dev[]");
        if (shard_total[g] && !shard_ptr[g]) return fail_arg("null shard");
        pos[(size_t)g] = acc; acc += shard_total[g];
        if (shard_pos) shard_pos[g] = pos[(size_t)g];
    }
    if (acc > dst_capacity) return fail_arg("dst_capacity must hold the sum of shard_total[]");
    int my_cuda_device = -1;
    if (cudaGetDevice(&my_cuda_device) != cudaSuccess) my_cuda_device = -1;
    // one copy per shard, each on a stream of its SOURCE device, so the links into dst_dev are all busy at once
    std::vector<cudaStream_t> st((size_t)nshard, nullptr);
    cudaError_t err = cudaSuccess; const char* where = "";
    for (int g = 0; g < nshard && err == cudaSuccess; g++) {
        if (!shard_total[g]) continue;
        if ((err = cudaSetDevice(shard_dev[g])) != cudaSuccess) { where = "cudaSetDevice"; break; }
        if (shard_dev[g] != dst_dev) {
            int can = 0;
            if (cudaDeviceCanAccessPeer(&can, shard_dev[g], dst_dev) == cudaSuccess && can) {
                const cudaError_t e = cudaDeviceEnablePeerAccess(dst_dev, 0);        // direct NVLink/PCIe stores; without it the copy is staged
                if (e != cudaSuccess) (void)cudaGetLastError();                      // (already enabled, or not possible: either way the copy below works)
            }
        }
        if ((err = cudaStreamCreateWithFlags(&st[(size_t)g], cudaStreamNonBlocking)) != cudaSuccess) { st[(size_t)g] = nullptr; where = "cudaStreamCreate"; break; }
        uint8_t* to = (uint8_t*)dst + pos[(size_t)g];
        err = shard_dev[g] == dst_dev ? cudaMemcpyAsync(to, shard_ptr[g], shard_total[g], cudaMemcpyDeviceToDevice, st[(size_t)g])
                                      : cudaMemcpyPeerAsync(to, dst_dev, shard_ptr[g], shard_dev[g], shard_total[g], st[(size_t)g]);
        where = "peer copy";
    }
    for (int g = 0; g < nshard; g++) {
        if (!st[(size_t)g]) continue;
        cudaSetDevice(shard_dev[g]);
        const cudaError_t e = cudaStreamSynchronize(st[(size_t)g]);
        if (err == cudaSuccess && e != cudaSuccess) { err = e; where = "cudaStreamSynchronize"; }
        cudaStreamDestroy(st[(size_t)g]);
    }
    if (my_cuda_device >= 0) cudaSetDevice(my_cuda_device);
    if (err != cudaSuccess) return fail_cuda(err, where);
    return 0;
}

// ---- host-buffer batches
int b200lz4_compress_fast_batch_host(const uint8_t* src_base, const uint64_t* src_off, const int32_t* src_len,
                                     uint8_t* dst_base, const uint64_t* dst_off, const int32_t* dst_cap,
                                     int32_t* result, size_t n, int max_src_len)
{ return host_batch(OP_COMPRESS_FAST, src_base, src_off, src_len, dst_base, dst_off, dst_cap, result, n, max_src_len); }
int b200lz4_compress_hc_batch_host(const uint8_t* src_base, const uint64_t* src_off, const int32_t* src_len,
                                   uint8_t* dst_base, const uint64_t* dst_off, const int32_t* dst_cap,
                                   int32_t* result, size_t n, int level)
{ return host_batch(OP_COMPRESS_HC, src_base, src_off, src_len, dst_base, dst_off, dst_cap, result, n, level); }
int b200lz4_decompress_safe_batch_host(const uint8_t* src_base, const uint64_t* src_off, const int32_t* src_len,
                                       uint8_t* dst_base, const uint64_t* dst_off, const int32_t* dst_cap,
                                       int32_t* result, size_t n)
{ return host_batch(OP_DEC_SAFE, src_base, src_off, src_len, dst_base, dst_off, dst_cap, result, n, 0); }
int b200lz4_decompress_fast_batch_host(const uint8_t* src_base, const uint64_t* src_off, const int32_t* src_avail,
                                       uint8_t* dst_base, const uint64_t* dst_off, const int32_t* dst_len,
                                       int32_t* result, size_t n)
{ return host_batch(OP_DEC_FAST, src_base, src_off, src_avail, dst_base, dst_off, dst_len, result, n, 0); }
int b200xxh32_batch_host(const uint8_t* base, const uint64_t* off, const int32_t* len, uint32_t seed, uint32_t* out, size_t n)
{ return hash_host_batch<uint32_t>(32, base, off, len, seed, out, n); }
int b200xxh64_batch_host(const uint8_t* base, const uint64_t* off, const int32_t* len, uint64_t seed, uint64_t* out, size_t n)
{ return hash_host_batch<uint64_t>(64, base, off, len, seed, out, n); }

int b200lz4_compress_fast_compact_host(const uint8_t* src_base, const uint64_t* src_off, const int32_t* src_len,
                                       uint8_t* dst_base, size_t dst_capacity, uint64_t* out_off,
                                       int32_t* result, size_t n, int max_src_len, uint64_t* total)
{
    if (total) *total = 0;
    if (n == 0) return 0;
    if (!src_base || !src_off || !src_len || !dst_base || !out_off || !result) return fail_arg("null pointer");
    // stage: each block gets a bound-sized slot in d_dst, launch_compact packs the results into d_aux
    auto stage = [&](Slot& s, const Chunk& ch) -> int {
        uint64_t bound_sum = 0;
        for (size_t k = ch.i0; k < ch.i0 + ch.nb; k++) bound_sum += aligned_compress_bound((uint64_t)(src_len[k] > 0 ? src_len[k] : 0));
        int rc = slot_reserve(s, ch.s_span + 16, (size_t)bound_sum + 16, ch.nb, (size_t)bound_sum + 16); if (rc) return rc;
        const size_t s_phase = (size_t)((uintptr_t)(src_base + ch.s_lo) & 15);
        uint64_t slot_pos = 0;
        for (size_t k = 0; k < ch.nb; k++) {
            const uint64_t len = (uint64_t)(src_len[ch.i0 + k] > 0 ? src_len[ch.i0 + k] : 0);
            s.h.soff()[k] = src_off[ch.i0 + k] - ch.s_lo + s_phase;
            s.h.doff()[k] = slot_pos;
            s.h.slen()[k] = src_len[ch.i0 + k];
            s.h.dcap()[k] = (int32_t)compress_bound(len);
            slot_pos += aligned_compress_bound(len);
        }
        CK(cudaMemcpyAsync(s.d.base, s.h.base, s.h.bytes(), cudaMemcpyHostToDevice, s.st));
        if (ch.s_span) CK(cudaMemcpyAsync(s.d_src + s_phase, src_base + ch.s_lo, ch.s_span, cudaMemcpyHostToDevice, s.st));
        BatchArgs a{ s.d_src, s.d.soff(), s.d.slen(), s.d_dst, s.d.doff(), s.d.dcap(), s.d.res(), ch.nb };
        CK(launch_op(OP_COMPRESS_FAST, a, max_src_len, s.st));
        g_launch_count.fetch_add(2, std::memory_order_relaxed);
        CK(launch_compact(s.d_dst, s.d.doff(), s.d.res(), s.d_aux, s.d.out(), s.d.total(), ch.nb, s.st));
        CK(cudaMemcpyAsync(s.h.base, s.d.base, s.h.bytes(), cudaMemcpyDeviceToHost, s.st));
        return 0;
    };
    // retire: learn the chunk's packed size, start the payload copy at the running offset
    uint64_t running = 0;
    auto retire = [&](Slot& s) -> int {
        const uint64_t tot = *s.h.total();
        if (running + tot > dst_capacity) return fail_arg("dst_capacity too small for the packed stream");
        if (tot) CK(cudaMemcpyAsync(dst_base + running, s.d_aux, (size_t)tot, cudaMemcpyDeviceToHost, s.st));
        CK(cudaEventRecord(s.drained, s.st)); s.draining = true;
        const size_t nb = s.i1 - s.i0;
        memcpy(result + s.i0, s.h.res(), nb * sizeof(int32_t));
        for (size_t k = 0; k < nb; k++) out_off[s.i0 + k] = running + s.h.out()[k];
        running += tot;
        return 0;
    };
    const int rc = run_pipeline(n, src_off, src_len, nullptr, nullptr, "blocks must ascend", stage, retire);
    if (!rc && total) *total = running;
    return rc;
}

int b200lz4_compress_fast_batch_host_multi(const uint8_t* src_base, const uint64_t* src_off, const int32_t* src_len,
                                           uint8_t* dst_base, const uint64_t* dst_off, const int32_t* dst_cap,
                                           int32_t* result, size_t n, int max_src_len, const int* devices, int ndev)
{ return multi_host_batch(OP_COMPRESS_FAST, src_base, src_off, src_len, dst_base, dst_off, dst_cap, result, n, max_src_len, devices, ndev); }
int b200lz4_compress_hc_batch_host_multi(const uint8_t* src_base, const uint64_t* src_off, const int32_t* src_len,
                                         uint8_t* dst_base, const uint64_t* dst_off, const int32_t* dst_cap,
                                         int32_t* result, size_t n, int level, const int* devices, int ndev)
{ return multi_host_batch(OP_COMPRESS_HC, src_base, src_off, src_len, dst_base, dst_off, dst_cap, result, n, level, devices, ndev); }
int b200lz4_decompress_safe_batch_host_multi(const uint8_t* src_base, const uint64_t* src_off, const int32_t* src_len,
                                             uint8_t* dst_base, const uint64_t* dst_off, const int32_t* dst_cap,
                                             int32_t* result, size_t n, const int* devices, int ndev)
{ return multi_host_batch(OP_DEC_SAFE, src_base, src_off, src_len, dst_base, dst_off, dst_cap, result, n, 0, devices, ndev); }
int b200lz4_decompress_fast_batch_host_multi(const uint8_t* src_base, const uint64_t* src_off, const int32_t* src_avail,
                                             uint8_t* dst_base, const uint64_t* dst_off, const int32_t* dst_len,
                                             int32_t* result, size_t n, const int* devices, int ndev)
{ return multi_host_batch(OP_DEC_FAST, src_base, src_off, src_avail, dst_base, dst_off, dst_len, result, n, 0, devices, ndev); }
int b200lz4_compress_fast_compact_host_multi(const uint8_t* src_base, const uint64_t* src_off, const int32_t* src_len,
                                             uint8_t* dst_base, size_t dst_capacity, uint64_t* out_off,
                                             int32_t* result, size_t n, int max_src_len, const int* devices, int ndev,
                                             uint64_t* shard_base, uint64_t* shard_total)
{
    if (ndev < 1 || ndev > 64) return fail_arg("ndev must be 1..64");
    for (int g = 0; g < ndev; g++) { if (shard_base) shard_base[g] = 0; if (shard_total) shard_total[g] = 0; }
    if (n == 0) return 0;
    if (!src_base || !src_off || !src_len || !dst_base || !out_off || !result) return fail_arg("null pointer");
    // region of shard g: the aligned bounds of its blocks, laid end to end (prefix sums at the shard boundaries only)
    std::vector<uint64_t> base((size_t)ndev + 1, 0);
    {
        uint64_t acc = 0; int g = 0;
        for (size_t i = 0; i <= n; i++) {
            while (g <= ndev && i == n * (size_t)g / (size_t)ndev) base[(size_t)g++] = acc;
            if (i < n) acc += aligned_compress_bound((uint64_t)(src_len[i] > 0 ? src_len[i] : 0));
        }
        if (acc > dst_capacity) return fail_arg("dst_capacity must hold the aligned bounds of all blocks");
    }
    return run_sharded(n, devices, ndev, [&](size_t lo, size_t cnt) {
        int g = 0;
        while (n * (size_t)(g + 1) / (size_t)ndev <= lo) g++;                  // which shard this range is
        uint64_t total = 0;
        int rc = b200lz4_compress_fast_compact_host(src_base, src_off + lo, src_len + lo, dst_base + base[(size_t)g],
                                                    (size_t)(base[(size_t)g + 1] - base[(size_t)g]), out_off + lo, result + lo, cnt,
                                                    max_src_len, &total);
        if (rc) return rc;
        for (size_t i = lo; i < lo + cnt; i++) out_off[i] += base[(size_t)g];
        if (shard_base) shard_base[g] = base[(size_t)g];
        if (shard_total) shard_total[g] = total;
        return 0;
    });
}
int b200xxh32_batch_host_multi(const uint8_t* base, const uint64_t* off, const int32_t* len, uint32_t seed,
                               uint32_t* out, size_t n, const int* devices, int ndev)
{
    if (n == 0) return 0;
    if (!base || !off || !len || !out) return fail_arg("null pointer");
    return run_sharded(n, devices, ndev, [&](size_t lo, size_t cnt) { return hash_host_batch<uint32_t>(32, base, off + lo, len + lo, seed, out + lo, cnt); });
}
int b200xxh64_batch_host_multi(const uint8_t* base, const uint64_t* off, const int32_t* len, uint64_t seed,
                               uint64_t* out, size_t n, const int* devices, int ndev)
{
    if (n == 0) return 0;
    if (!base || !off || !len || !out) return fail_arg("null pointer");
    return run_sharded(n, devices, ndev, [&](size_t lo, size_t cnt) { return hash_host_batch<uint64_t>(64, base, off + lo, len + lo, seed, out + lo, cnt); });
}

int b200lz4_context_count(void) { return g_contexts.load(std::memory_order_relaxed); }
uint64_t b200lz4_launch_count(void) { return g_launch_count.load(std::memory_order_relaxed); }
void     b200lz4_launch_count_reset(void) { g_launch_count.store(0, std::memory_order_relaxed); }

} // extern "C"
