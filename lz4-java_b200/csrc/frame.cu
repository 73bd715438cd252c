// frame.cu — LZ4 Frame batch decoder: LZ4FrameInputStream semantics (reference:
// src/java/net/jpountz/lz4/LZ4FrameInputStream.java:132-321; format src/lz4/doc/lz4_Frame_format.md)
// for a buffer holding any number of concatenated frames (skippable frames included).
//
// The stream adapter in the reference is strictly sequential: one block in flight, one XXH32 state per
// frame.  Here the host only INDEXES the container (magic / FLG / BD / block sizes: O(#blocks), no
// payload byte is touched), and the payload work is three batched launches on the device:
//   1. XXH32 over every frame descriptor (header checksum byte) and, if present, every block payload
//      (block checksums)                                            -> xxh_batch_kernel<32>
//   2. safe-decompress of every compressed block into its slot; stored blocks are copied
//                                                                   -> lz4_decompress_safe_kernel, gather
//   3. XXH32 over every frame's decoded content (content checksum)  -> xxh32_frames_chained_kernel: one warp per frame,
//      beside the decoder on a second stream, taking each block as soon as it is decoded
// Blocks of one frame are decoded in parallel because lz4-java only writes independent blocks
// (LZ4FrameOutputStream.java:58,361-363; dependent blocks are rejected like the reference does).
// With the container in device memory (b200lz4f_index_create_dev, b200lz4f_decompress_dev) the index pass itself runs on the
// device (frame_index.cu) and only its records come to the host; both indexers run the same walk (walk_frames, kernels.h).
#include "../../include/b200lz4.h"
#include "kernels.h"
#ifdef B200_HOST_SIM            // the emulator build compiles the host layer only: the device indexer's kernels come with it
#include "frame_index.cu"
#endif
#include <algorithm>
#include <cstring>
#include <new>
#include <vector>

namespace b200 {

cudaError_t launch_gather(const uint8_t* src, const uint64_t* src_off, const int32_t* lens,
                          uint8_t* dst, const uint64_t* dst_off, size_t n, cudaStream_t st);

struct FrameRec {
    uint64_t desc_off; int32_t desc_len; uint8_t hc_byte; uint8_t flg; uint32_t bs;
    uint64_t content_size; bool has_size;
    size_t first_block, nblocks;
    uint32_t content_checksum; bool has_checksum;
    uint64_t out_off;                   // slot-layout start of this frame's content
    bool complete;                      // read up to its EndMark (and content checksum); false: the container breaks off inside it
};

struct BlockRec { uint64_t src_off; uint32_t size; bool raw; uint32_t checksum; bool has_checksum; size_t frame; uint64_t out_off; uint32_t cap; };

struct FrameIndex {
    std::vector<FrameRec> frames;
    std::vector<BlockRec> blocks;
    uint64_t slot_bytes = 0;            // device bytes needed for the slot layout (upper bound of the decoded size)
    int tail_err = 0;                   // the container's own error, behind everything indexed (reported after what precedes it)
    // device-side descriptor arrays, built once
    int device = -1;
    uint8_t* d_blob = nullptr; size_t blob_bytes = 0;
    std::vector<uint8_t> h_blob;
    // offsets inside the blob
    size_t o_c_soff, o_c_doff, o_c_slen, o_c_dcap, o_c_res;          // compressed blocks
    size_t o_r_soff, o_r_doff, o_r_len;                              // raw blocks
    size_t o_h_off, o_h_len, o_h_out;                                // header descriptors
    size_t o_b_off, o_b_len, o_b_out;                                // block checksums
    size_t o_f_first, o_f_nblk, o_f_out;                                        // content checksums (chained to the decoder: xxhash.cu)
    size_t o_k_comp, o_k_rawlen, o_k_off;                            // per block: index among the compressed blocks (-1: stored), stored size, slot
    cudaStream_t st2 = nullptr; cudaEvent_t e1 = nullptr, e2 = nullptr;   // the checksum warps run beside the decoder
    size_t n_comp = 0, n_raw = 0, n_bsum = 0, n_fsum = 0;
    std::vector<size_t> comp_ix, raw_ix, bsum_ix, fsum_ix;
};

// The host sink of walk_frames (kernels.h): frames and blocks into the index, each block with its slot.  The device indexer
// replays its walkers' records through it, so both indexers lay out slots the same way.
struct IndexSink {
    FrameIndex& ix; FrameRec f{};
    void frame_begin(const WalkFrame& w)
    {
        f = FrameRec{};
        f.desc_off = w.desc_off; f.desc_len = w.desc_len; f.hc_byte = w.hc_byte; f.flg = w.flg;
        f.bs = 1u << (8 + 2 * (w.bd >> 4));
        f.first_block = ix.blocks.size();
        f.out_off = ix.slot_bytes;
    }
    void block(uint64_t src_off, uint32_t word, uint32_t checksum)
    {
        BlockRec b{}; b.src_off = src_off; b.size = word & 0x7FFFFFFFu; b.raw = word >> 31; b.frame = ix.frames.size();
        b.has_checksum = f.flg & 0x10;
        if (b.has_checksum) b.checksum = checksum;
        // the slot: a stored block needs its own size, a compressed one cannot decode to more than 255 bytes per byte
        // (one length byte adds at most 255) -- so a stream of tiny flushed blocks asks for what it can fill, not for
        // blockMaxSize each.  Full blocks keep exactly bs: a frame without short blocks in the middle stays contiguous.
        const uint64_t room = b.raw ? b.size : std::min<uint64_t>(f.bs, 255ull * b.size);
        b.cap = (uint32_t)room;
        b.out_off = ix.slot_bytes; ix.slot_bytes += room >= f.bs ? f.bs : ((room + 15) & ~15ull);
        ix.blocks.push_back(b);
    }
    void frame_end(const WalkFrame& w)
    {
        f.nblocks = ix.blocks.size() - f.first_block;
        f.content_size = w.content_size; f.has_size = w.has_size;
        f.content_checksum = w.content_checksum; f.has_checksum = w.has_checksum;
        f.complete = w.complete;
        ix.frames.push_back(f);
    }
};

// What the whole container's walk means for the index.  The reader is a stream: it hands out the bytes of every frame before
// a malformed spot and fails THERE, after any checksum or decode error that lies earlier.  So an error behind at least one
// indexed frame is not returned here: it is kept in ix.tail_err, what precedes it is decoded and verified like any other
// input (the blocks of a frame cut short included -- that frame has no content checks), and decode_dev reports the first
// error in stream order.
static int index_verdict(FrameIndex& ix, int err, bool seen)
{
    if (err) {
        if (ix.frames.empty()) return err;                                      // nothing lies before the error
        ix.tail_err = err;
        return 0;
    }
    return seen ? 0 : -1;
}

// LZ4FrameInputStream.nextFrameInfo / readHeader / readBlock as a pure index pass over host memory
static int index_frames(const uint8_t* src, size_t n, FrameIndex& ix, bool single = false, size_t* consumed = nullptr)
{
    IndexSink sink{ ix };
    const WalkEnd e = walk_frames(src, n, 0, n, single, sink);
    if (consumed) *consumed = e.ip;
    return index_verdict(ix, e.err, e.seen);
}

// ---- the same index from bytes in device memory (walkers: frame_index.cu).  Only records come back, never payload.
// Where the arrays of one walk with m walkers lie, the same in d_seg and h_seg: the segments go up, the rest comes back.
struct WalkLayout {
    size_t segs, sums, lens, pos, total, bytes = 0;
    explicit WalkLayout(size_t m)
    {
        auto take = [&](size_t n) { const size_t at = bytes; bytes = (bytes + n + 15) & ~size_t(15); return at; };
        segs = take(sizeof(WalkSeg) * m); sums = take(sizeof(WalkSummary) * m); lens = take(4 * m); pos = take(8 * m); total = take(16);
    }
};
static constexpr uint64_t WALK_MAX_REC = 0x7FFFFFFFull;      // records of one walker (the packing scan counts in int32)

// One walker per segment: summaries into sum[], the records each walker wrote appended to recs (walker j's from rec_at[j]).
// A region guess that proved too small is run once more, for those walkers only, with room for exactly what they counted.
static int walk_segments(FrameReadScratch& s, const uint8_t* d_src, uint64_t n, bool single, const uint64_t* start, const uint64_t* end,
                         size_t m, WalkSummary* sum, uint64_t* rec_at, std::vector<WalkRec>& recs, cudaStream_t st)
{
    std::vector<size_t> todo(m);
    std::vector<uint64_t> cap(m);
    for (size_t j = 0; j < m; j++) { todo[j] = j; cap[j] = std::min(((end[j] - start[j]) >> 12) + 64, WALK_MAX_REC); }   // ~ one per 4 KiB
#define WCK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) return fail_cuda(e_, #call); } while (0)
    while (!todo.empty()) {
        const size_t k = todo.size();
        const WalkLayout L(k);
        uint64_t room = 0;
        for (size_t i = 0; i < k; i++) room += cap[todo[i]];
        int rc = reserve_device(s.d_seg, s.seg_cap, L.bytes);
        if (!rc) rc = reserve_pinned(s.h_seg, s.h_seg_cap, std::max<size_t>(L.bytes, room * sizeof(WalkRec)));
        if (!rc) rc = reserve_device(s.d_recs, s.recs_cap, room * sizeof(WalkRec) + 16);
        if (!rc) rc = reserve_device(s.d_packed, s.packed_cap, room * sizeof(WalkRec) + 16);
        if (rc) return rc;
        WalkSeg* hs = (WalkSeg*)(s.h_seg + L.segs);
        uint64_t at = 0;
        for (size_t i = 0; i < k; i++) { const size_t j = todo[i]; hs[i] = WalkSeg{ start[j], end[j], at, cap[j] }; at += cap[j]; }
        uint8_t* D = s.d_seg;
        WCK(cudaMemcpyAsync(D, s.h_seg, L.sums, cudaMemcpyHostToDevice, st));
        g_launch_count.fetch_add(3, std::memory_order_relaxed);
        WCK(launch_frame_walk(d_src, n, single, (const WalkSeg*)D, (WalkSummary*)(D + L.sums), (int32_t*)(D + L.lens), (WalkRec*)s.d_recs, (uint32_t)k, st));
        WCK(launch_scan((const int32_t*)(D + L.lens), (uint64_t*)(D + L.pos), (uint64_t*)(D + L.total), nullptr, k, st));
        WCK(launch_frame_pack((const WalkSeg*)D, (const int32_t*)(D + L.lens), (const uint64_t*)(D + L.pos), (const WalkRec*)s.d_recs,
                              (WalkRec*)s.d_packed, (uint32_t)k, st));
        WCK(cudaMemcpyAsync(s.h_seg + L.sums, D + L.sums, L.bytes - L.sums, cudaMemcpyDeviceToHost, st));
        WCK(cudaStreamSynchronize(st));
        const uint64_t packed = *(const uint64_t*)(s.h_seg + L.total);
        const WalkSummary* hsum = (const WalkSummary*)(s.h_seg + L.sums);
        const uint64_t* hpos = (const uint64_t*)(s.h_seg + L.pos);
        std::vector<WalkSummary> got(hsum, hsum + k);
        std::vector<uint64_t> pos(hpos, hpos + k);
        if (packed) {
            WCK(cudaMemcpyAsync(s.h_seg, s.d_packed, packed * sizeof(WalkRec), cudaMemcpyDeviceToHost, st));
            WCK(cudaStreamSynchronize(st));
        }
        const size_t base = recs.size();
        recs.insert(recs.end(), (const WalkRec*)s.h_seg, (const WalkRec*)s.h_seg + packed);
        std::vector<size_t> again;
        for (size_t i = 0; i < k; i++) {
            const size_t j = todo[i];
            sum[j] = got[i]; rec_at[j] = base + pos[i];
            if (got[i].nrec > cap[j]) {
                if (got[i].nrec > WALK_MAX_REC) return fail_arg("more than 2^31 frames and blocks between two frame hints");
                cap[j] = got[i].nrec; again.push_back(j);
            }
        }
        todo.swap(again);
    }
#undef WCK
    return 0;
}

// walker records -> the index, through the host indexer's own sink (records: frame_index.cu, RecordSink)
static void replay(const WalkRec* r, uint64_t nrec, IndexSink& sink)
{
    for (uint64_t i = 0; i + 2 <= nrec;) {
        WalkFrame f{};
        const uint32_t bits = (uint32_t)(r[i + 1].b >> 32);
        f.desc_off = r[i].a; f.content_size = r[i].b; f.nblocks = r[i + 1].a; f.content_checksum = (uint32_t)r[i + 1].b;
        f.flg = (uint8_t)bits; f.bd = (uint8_t)(bits >> 8); f.hc_byte = (uint8_t)(bits >> 16); f.desc_len = (uint8_t)((bits >> 24) & 15);
        f.complete = bits & (1u << 28); f.has_checksum = bits & (1u << 29); f.has_size = bits & (1u << 30);
        i += 2;
        sink.frame_begin(f);
        for (uint64_t k = 0; k < f.nblocks; k++, i++) sink.block(r[i].a, (uint32_t)r[i].b, (uint32_t)(r[i].b >> 32));
        sink.frame_end(f);
    }
}

// The chain of the container from offset 0, stitched from walkers that started at the hints.  Where it does not land on a
// hint, a walker is run from where it is to the next hint: a wrong hint costs a launch, never a different index.
static int index_frames_dev(FrameReadScratch& s, const uint8_t* d_src, uint64_t n, bool single, const uint64_t* hint, size_t nhint,
                            FrameIndex& ix, size_t* consumed, cudaStream_t st)
{
    const size_t m = nhint + 1;
    std::vector<uint64_t> start(m), end(m), rec_at(m);
    start[0] = 0;
    for (size_t j = 0; j < nhint; j++) { end[j] = hint[j]; start[j + 1] = hint[j]; }
    end[nhint] = n;
    std::vector<WalkSummary> sum(m);
    std::vector<WalkRec> recs;
    int rc = walk_segments(s, d_src, n, single, start.data(), end.data(), m, sum.data(), rec_at.data(), recs, st);
    if (rc) return rc;
    IndexSink sink{ ix };
    WalkSummary cur = sum[0]; uint64_t cur_at = rec_at[0];
    size_t next = 1;
    bool seen = false;
    for (;;) {
        replay(recs.data() + cur_at, cur.nrec, sink);
        seen |= cur.flags & WALK_SEEN;
        if (cur.err || (cur.flags & WALK_SINGLE_DONE) || cur.ip >= n) break;
        while (next < m && start[next] < cur.ip) next++;
        if (next < m && start[next] == cur.ip) { cur = sum[next]; cur_at = rec_at[next]; next++; continue; }
        const uint64_t from = cur.ip, to = next < m ? start[next] : n;
        rc = walk_segments(s, d_src, n, single, &from, &to, 1, &cur, &cur_at, recs, st);
        if (rc) return rc;
    }
    if (consumed) *consumed = cur.ip;
    return index_verdict(ix, cur.err, seen);
}

// Packs decoded blocks back to back: block b's blen[b] bytes move from d_slots + its slot to d_dst + the lengths before it.
// d_desc: device room for pack_desc_bytes(blocks) of descriptors.  One launch; ordered on st.
static size_t pack_desc_bytes(size_t nb) { return 2 * ((nb * 8 + 15) & ~size_t(15)) + nb * 4; }
static cudaError_t pack_blocks(const FrameIndex& ix, const int32_t* blen, const uint8_t* d_slots, uint8_t* d_dst, uint8_t* d_desc, cudaStream_t st)
{
    const size_t nb = ix.blocks.size();
    if (nb == 0) return cudaSuccess;
    const size_t o_to = (nb * 8 + 15) & ~size_t(15), o_len = 2 * o_to;
    std::vector<uint8_t> h(pack_desc_bytes(nb));
    uint64_t pos = 0;
    for (size_t b = 0; b < nb; b++) {
        ((uint64_t*)h.data())[b] = ix.blocks[b].out_off;
        ((uint64_t*)(h.data() + o_to))[b] = pos; pos += (uint64_t)blen[b];
    }
    memcpy(h.data() + o_len, blen, nb * 4);
    const cudaError_t e = cudaMemcpyAsync(d_desc, h.data(), h.size(), cudaMemcpyHostToDevice, st);   // pageable: staged before it returns
    if (e != cudaSuccess) return e;
    g_launch_count += 1;
    return launch_gather(d_slots, (const uint64_t*)d_desc, (const int32_t*)(d_desc + o_len), d_dst, (const uint64_t*)(d_desc + o_to), nb, st);
}

template <typename T> static size_t put(std::vector<uint8_t>& blob, size_t count)
{
    size_t o = (blob.size() + 15) & ~size_t(15);
    blob.resize(o + count * sizeof(T));
    return o;
}

static int build_descriptors(FrameIndex& ix)
{
    for (size_t i = 0; i < ix.blocks.size(); i++) {
        (ix.blocks[i].raw ? ix.raw_ix : ix.comp_ix).push_back(i);
        if (ix.blocks[i].has_checksum) ix.bsum_ix.push_back(i);
    }
    for (size_t f = 0; f < ix.frames.size(); f++) if (ix.frames[f].has_checksum) ix.fsum_ix.push_back(f);
    ix.n_comp = ix.comp_ix.size(); ix.n_raw = ix.raw_ix.size(); ix.n_bsum = ix.bsum_ix.size(); ix.n_fsum = ix.fsum_ix.size();
    auto& B = ix.h_blob;
    const size_t nf = ix.frames.size();
    ix.o_c_soff = put<uint64_t>(B, ix.n_comp); ix.o_c_doff = put<uint64_t>(B, ix.n_comp);
    ix.o_c_slen = put<int32_t>(B, ix.n_comp);  ix.o_c_dcap = put<int32_t>(B, ix.n_comp); ix.o_c_res = put<int32_t>(B, ix.n_comp);
    ix.o_r_soff = put<uint64_t>(B, ix.n_raw);  ix.o_r_doff = put<uint64_t>(B, ix.n_raw); ix.o_r_len = put<int32_t>(B, ix.n_raw);
    ix.o_h_off = put<uint64_t>(B, nf); ix.o_h_len = put<int32_t>(B, nf); ix.o_h_out = put<uint32_t>(B, nf);
    ix.o_b_off = put<uint64_t>(B, ix.n_bsum); ix.o_b_len = put<int32_t>(B, ix.n_bsum); ix.o_b_out = put<uint32_t>(B, ix.n_bsum);
    ix.o_f_first = put<uint32_t>(B, ix.n_fsum); ix.o_f_nblk = put<uint32_t>(B, ix.n_fsum); ix.o_f_out = put<uint32_t>(B, ix.n_fsum);
    ix.o_k_comp = put<int32_t>(B, ix.blocks.size()); ix.o_k_rawlen = put<int32_t>(B, ix.blocks.size());
    ix.o_k_off = put<uint64_t>(B, ix.blocks.size());
    B.resize((B.size() + 15) & ~size_t(15));
    uint8_t* p = B.data();
    for (size_t k = 0; k < ix.blocks.size(); k++) ((uint64_t*)(p + ix.o_k_off))[k] = ix.blocks[k].out_off;
    for (size_t k = 0; k < ix.n_comp; k++) ((int32_t*)(p + ix.o_k_comp))[ix.comp_ix[k]] = (int32_t)k;
    for (size_t k = 0; k < ix.n_raw; k++) { ((int32_t*)(p + ix.o_k_comp))[ix.raw_ix[k]] = -1; ((int32_t*)(p + ix.o_k_rawlen))[ix.raw_ix[k]] = (int32_t)ix.blocks[ix.raw_ix[k]].size; }
    for (size_t k = 0; k < ix.n_fsum; k++) {
        const FrameRec& fr = ix.frames[ix.fsum_ix[k]];
        if (fr.first_block > 0xFFFFFFFFull || fr.nblocks > 0xFFFFFFFFull) return -10;
        ((uint32_t*)(p + ix.o_f_first))[k] = (uint32_t)fr.first_block; ((uint32_t*)(p + ix.o_f_nblk))[k] = (uint32_t)fr.nblocks;
    }
    for (size_t k = 0; k < ix.n_comp; k++) {
        const BlockRec& b = ix.blocks[ix.comp_ix[k]];
        ((uint64_t*)(p + ix.o_c_soff))[k] = b.src_off; ((uint64_t*)(p + ix.o_c_doff))[k] = b.out_off;
        ((int32_t*)(p + ix.o_c_slen))[k] = (int32_t)b.size; ((int32_t*)(p + ix.o_c_dcap))[k] = (int32_t)b.cap;
    }
    for (size_t k = 0; k < ix.n_raw; k++) {
        const BlockRec& b = ix.blocks[ix.raw_ix[k]];
        ((uint64_t*)(p + ix.o_r_soff))[k] = b.src_off; ((uint64_t*)(p + ix.o_r_doff))[k] = b.out_off; ((int32_t*)(p + ix.o_r_len))[k] = (int32_t)b.size;
    }
    for (size_t f = 0; f < nf; f++) { ((uint64_t*)(p + ix.o_h_off))[f] = ix.frames[f].desc_off; ((int32_t*)(p + ix.o_h_len))[f] = ix.frames[f].desc_len; }
    for (size_t k = 0; k < ix.n_bsum; k++) {
        const BlockRec& b = ix.blocks[ix.bsum_ix[k]];
        ((uint64_t*)(p + ix.o_b_off))[k] = b.src_off; ((int32_t*)(p + ix.o_b_len))[k] = (int32_t)b.size;
    }
    return 0;
}

} // namespace b200

using namespace b200;

extern "C" {

static void* index_create(const uint8_t* src_host, size_t n, bool single, uint64_t* slot_bytes, size_t* consumed, int* err)
{
    FrameIndex* ix = new (std::nothrow) FrameIndex();
    if (!ix) { if (err) *err = B200LZ4_E_ARG; return nullptr; }
    int rc = src_host ? index_frames(src_host, n, *ix, single, consumed) : -1;
    if (rc == 0) rc = build_descriptors(*ix);
    if (rc) { delete ix; if (err) *err = rc; return nullptr; }
    if (slot_bytes) *slot_bytes = ix->slot_bytes;
    if (err) *err = 0;
    return ix;
}

void* b200lz4f_index_create(const uint8_t* src_host, size_t n, uint64_t* slot_bytes, int* err)
{ return index_create(src_host, n, false, slot_bytes, nullptr, err); }
void* b200lz4f_index_create_single(const uint8_t* src_host, size_t n, uint64_t* slot_bytes, size_t* src_consumed, int* err)
{ return index_create(src_host, n, true, slot_bytes, src_consumed, err); }

void* b200lz4f_index_create_dev(const uint8_t* d_src, size_t n, int single, const uint64_t* frame_hint, size_t nhint,
                                uint64_t* slot_bytes, size_t* src_consumed, int* err, void* stream)
{
    auto fail = [&](int rc) -> void* { if (err) *err = rc; return nullptr; };
    if (nhint && !frame_hint) return fail(fail_arg("frame_hint is NULL"));
    for (size_t j = 0; j < nhint; j++)
        if (frame_hint[j] >= n || (j && frame_hint[j] < frame_hint[j - 1])) return fail(fail_arg("frame hints must be ascending and below srcSize"));
    if (n && !d_src) return fail(fail_arg("null pointer"));
    if (n == 0) { if (src_consumed) *src_consumed = 0; return fail(-1); }      // no frame at all, like index_create
    FrameReadScratch* s;
    int rc = get_frame_read_scratch(&s);
    if (rc) return fail(rc);
    FrameIndex* ix = new (std::nothrow) FrameIndex();
    if (!ix) return fail(fail_arg("out of host memory"));
    const cudaStream_t st = (cudaStream_t)stream;
    rc = index_frames_dev(*s, d_src, n, single != 0, frame_hint, nhint, *ix, src_consumed, st);
    if (rc == B200LZ4_E_CUDA) cudaStreamSynchronize(st);                        // a failed call leaves nothing running on the scratch
    if (rc == 0) rc = build_descriptors(*ix);
    if (rc) { delete ix; return fail(rc); }
    if (slot_bytes) *slot_bytes = ix->slot_bytes;
    if (err) *err = 0;
    return ix;
}

// getExpectedContentSize / isExpectedContentSizeDefined (:416-445): the content size the first non-skippable frame declares,
// -1 when it declares none or when there is no frame at all; the descriptor hash is verified like nextFrameInfo does.
int b200lz4f_expected_content_size(const uint8_t* src, size_t n, int64_t* content_size)
{
    if (!src || !content_size) return B200LZ4_E_ARG;
    *content_size = -1;
    size_t ip = 0; bool seen = false;
    for (;;) {
        if (n - ip < 4) return (seen && n == ip) ? 0 : -1;                      // clean end behind skippable frames: "no frame" (:141-147)
        const uint32_t magic = rd32(src + ip); ip += 4;
        if ((magic >> 4) == (0x184D2A50u >> 4)) {
            if (n - ip < 4) return -1;
            const uint32_t sz = rd32(src + ip); ip += 4;
            if (n - ip < sz) return -1;
            ip += sz; seen = true; continue;
        }
        if (magic != 0x184D2204u) return -2;
        const size_t desc = ip;
        if (n - ip < 2) return -1;
        const uint8_t flg = src[ip++], bd = src[ip++];
        if ((flg >> 6) != 1 || (flg & 2) || !(flg & 0x20) || (flg & 1)) return -10;
        if ((bd & 0x8F) || (bd >> 4) < 4) return -10;
        uint64_t size = 0;
        if (flg & 8) { if (n - ip < 8) return -1; size = (uint64_t)rd32(src + ip) | ((uint64_t)rd32(src + ip + 4) << 32); ip += 8; }
        if (n - ip < 1) return -1;
        const uint32_t h = b200xxh32(src + desc, ip - desc, 0);
        const int st = b200lz4_last_status();
        if (st) return st;
        if (((h >> 8) & 0xFF) != src[ip]) return -3;
        if (flg & 8) *content_size = (int64_t)size;
        return 0;
    }
}

void b200lz4f_index_free(void* index)
{
    FrameIndex* ix = (FrameIndex*)index;
    if (!ix) return;
    if (ix->d_blob) { cudaSetDevice(ix->device); cudaFree(ix->d_blob); }
    if (ix->st2) { cudaSetDevice(ix->device); cudaStreamDestroy(ix->st2); cudaEventDestroy(ix->e1); cudaEventDestroy(ix->e2); }
    delete ix;
}

// Decode every indexed frame: d_src holds the container bytes, d_slots (>= slot_bytes) receives block b at its slot
// (b200lz4f_index_block_offsets; full blocks of one frame lie back to back).  On success frame_off[f] / frame_len[f] (host
// arrays, may be NULL) describe each frame's content, one run inside d_slots when no block was flushed short mid-frame;
// otherwise -11 is returned after every check has passed and the caller reads block by block (the host path below does).
// Returns total decoded bytes or a negative code.
int64_t b200lz4f_decode_dev(void* index, const uint8_t* d_src, uint8_t* d_slots, uint64_t* frame_off, uint64_t* frame_len,
                            int32_t* block_len_out, void* stream)
{
    FrameIndex& ix = *(FrameIndex*)index;
    cudaStream_t st = (cudaStream_t)stream;
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return B200LZ4_E_NODEVICE;
    if (ix.st2 && ix.device != dev) { cudaSetDevice(ix.device); cudaStreamDestroy(ix.st2); cudaEventDestroy(ix.e1); cudaEventDestroy(ix.e2); cudaSetDevice(dev); ix.st2 = nullptr; }
    if (!ix.d_blob || ix.device != dev) {
        if (ix.d_blob) { cudaSetDevice(ix.device); cudaFree(ix.d_blob); cudaSetDevice(dev); ix.d_blob = nullptr; }
        if (cudaMalloc(&ix.d_blob, ix.h_blob.size() + 16) != cudaSuccess) return B200LZ4_E_CUDA;
        ix.device = dev;
    }
    if (!ix.st2) {
        if (cudaStreamCreateWithFlags(&ix.st2, cudaStreamNonBlocking) != cudaSuccess) { ix.st2 = nullptr; return B200LZ4_E_CUDA; }
        if (cudaEventCreateWithFlags(&ix.e1, cudaEventDisableTiming) != cudaSuccess || cudaEventCreateWithFlags(&ix.e2, cudaEventDisableTiming) != cudaSuccess)
            return B200LZ4_E_CUDA;
    }
    uint8_t* D = ix.d_blob; uint8_t* H = ix.h_blob.data();
    const size_t nf = ix.frames.size();
    if (cudaMemcpyAsync(D, H, ix.h_blob.size(), cudaMemcpyHostToDevice, st) != cudaSuccess) return B200LZ4_E_CUDA;
    if (ix.n_comp && cudaMemsetAsync(D + ix.o_c_res, 0x80, ix.n_comp * 4, st) != cudaSuccess) return B200LZ4_E_CUDA;   // FRAME_RES_PENDING
    // 1. header + block checksums
    g_launch_count += 1;
    if (launch_xxh32(d_src, (uint64_t*)(D + ix.o_h_off), (int32_t*)(D + ix.o_h_len), 0, (uint32_t*)(D + ix.o_h_out), nf, st) != cudaSuccess) return B200LZ4_E_CUDA;
    if (ix.n_bsum) {
        // few long payloads: one warp per stream; many short ones: one lane per buffer (xxhash.cu)
        uint64_t sum = 0; for (size_t k = 0; k < ix.n_bsum; k++) sum += ix.blocks[ix.bsum_ix[k]].size;
        g_launch_count += 1;
        if ((sum / ix.n_bsum >= XXH_LONG_AVG ? launch_xxh32_long : launch_xxh32)(
                d_src, (uint64_t*)(D + ix.o_b_off), (int32_t*)(D + ix.o_b_len), 0, (uint32_t*)(D + ix.o_b_out), ix.n_bsum, st) != cudaSuccess) return B200LZ4_E_CUDA;
    }
    // 2. stored blocks are copied, then every compressed block is decoded; 3. one warp per frame folds the blocks into the
    // content checksum as the decoder hands them over (second stream; the decode kernel is launched FIRST and waits for nobody)
    if (ix.n_raw) {
        g_launch_count += 1;
        if (launch_gather(d_src, (uint64_t*)(D + ix.o_r_soff), (int32_t*)(D + ix.o_r_len), d_slots, (uint64_t*)(D + ix.o_r_doff), ix.n_raw, st) != cudaSuccess) return B200LZ4_E_CUDA;
    }
    if (cudaEventRecord(ix.e1, st) != cudaSuccess) return B200LZ4_E_CUDA;
    if (ix.n_comp) {
        BatchArgs a{ d_src, (uint64_t*)(D + ix.o_c_soff), (int32_t*)(D + ix.o_c_slen), d_slots, (uint64_t*)(D + ix.o_c_doff),
                     (int32_t*)(D + ix.o_c_dcap), (int32_t*)(D + ix.o_c_res), ix.n_comp };
        g_launch_count += 1;
        if (launch_decompress_safe(a, st) != cudaSuccess) return B200LZ4_E_CUDA;
    }
    if (ix.n_fsum) {
        if (cudaStreamWaitEvent(ix.st2, ix.e1, 0) != cudaSuccess) return B200LZ4_E_CUDA;
        g_launch_count += 1;
        if (launch_xxh32_frames_chained(d_slots, (uint64_t*)(D + ix.o_k_off), (uint32_t*)(D + ix.o_f_first), (uint32_t*)(D + ix.o_f_nblk),
                                        (int32_t*)(D + ix.o_k_comp), (int32_t*)(D + ix.o_k_rawlen),
                                        (int32_t*)(D + ix.o_c_res), (uint32_t*)(D + ix.o_f_out), ix.n_fsum, ix.st2) != cudaSuccess) return B200LZ4_E_CUDA;
        if (cudaEventRecord(ix.e2, ix.st2) != cudaSuccess || cudaStreamWaitEvent(st, ix.e2, 0) != cudaSuccess) return B200LZ4_E_CUDA;
    }
    if (ix.n_comp && cudaMemcpyAsync(H + ix.o_c_res, D + ix.o_c_res, ix.n_comp * 4, cudaMemcpyDeviceToHost, st) != cudaSuccess) return B200LZ4_E_CUDA;
    if (cudaMemcpyAsync(H + ix.o_h_out, D + ix.o_h_out, nf * 4, cudaMemcpyDeviceToHost, st) != cudaSuccess) return B200LZ4_E_CUDA;
    if (ix.n_bsum && cudaMemcpyAsync(H + ix.o_b_out, D + ix.o_b_out, ix.n_bsum * 4, cudaMemcpyDeviceToHost, st) != cudaSuccess) return B200LZ4_E_CUDA;
    if (ix.n_fsum && cudaMemcpyAsync(H + ix.o_f_out, D + ix.o_f_out, ix.n_fsum * 4, cudaMemcpyDeviceToHost, st) != cudaSuccess) return B200LZ4_E_CUDA;
    if (cudaStreamSynchronize(st) != cudaSuccess) return B200LZ4_E_CUDA;

    // the verdict, in the order the stream reader meets things: frame by frame -- descriptor hash (:208-216), then block by
    // block its checksum (:298-303) and its decode (:307-311), then at the EndMark content checksum (:266-269) and size (:270-272)
    std::vector<int32_t> bsum_of(ix.blocks.size(), -1), fsum_of(nf, -1);
    for (size_t k = 0; k < ix.n_bsum; k++) bsum_of[ix.bsum_ix[k]] = (int32_t)k;
    for (size_t k = 0; k < ix.n_fsum; k++) fsum_of[ix.fsum_ix[k]] = (int32_t)k;
    const int32_t* blk_comp = (const int32_t*)(H + ix.o_k_comp);
    std::vector<int32_t> blen(ix.blocks.size());
    int64_t total = 0; bool gaps = false;
    for (size_t f = 0; f < nf; f++) {
        const FrameRec& fr = ix.frames[f];
        if (((((uint32_t*)(H + ix.o_h_out))[f] >> 8) & 0xFF) != fr.hc_byte) return -3;
        uint64_t len = 0;
        for (size_t k = 0; k < fr.nblocks; k++) {
            const size_t b = fr.first_block + k;
            const BlockRec& br = ix.blocks[b];
            if (bsum_of[b] >= 0 && ((uint32_t*)(H + ix.o_b_out))[bsum_of[b]] != br.checksum) return -5;
            int32_t l = (int32_t)br.size;
            if (!br.raw) { l = ((int32_t*)(H + ix.o_c_res))[blk_comp[b]]; if (l < 0) return -6; }   // LZ4Exception -> IOException
            blen[b] = l;
            if (k + 1 < fr.nblocks && (uint32_t)l != fr.bs) gaps = true;          // a short block in the middle of a frame
            len += (uint64_t)l;
        }
        if (fsum_of[f] >= 0 && ((uint32_t*)(H + ix.o_f_out))[fsum_of[f]] != fr.content_checksum) return -7;
        if (fr.has_size && fr.content_size != len) return -8;
        if (frame_off) frame_off[f] = fr.out_off;
        if (frame_len) frame_len[f] = len;
        total += (int64_t)len;
    }
    if (ix.tail_err) return ix.tail_err;                    // the container breaks off / is malformed behind all that
    if (block_len_out) memcpy(block_len_out, blen.data(), blen.size() * sizeof(int32_t));
    return gaps ? -11 : total;                              // -11: everything verified, but read the blocks one by one
}

size_t b200lz4f_index_frames(void* index) { return ((FrameIndex*)index)->frames.size(); }
size_t b200lz4f_index_blocks(void* index) { return ((FrameIndex*)index)->blocks.size(); }
void b200lz4f_index_block_offsets(void* index, uint64_t* block_off)
{
    const FrameIndex& ix = *(FrameIndex*)index;
    for (size_t b = 0; b < ix.blocks.size(); b++) block_off[b] = ix.blocks[b].out_off;
}

// Whole thing with HOST buffers: index, upload, decode, download frame by frame into one contiguous stream.
static int64_t decompress_host(const uint8_t* src, size_t n, uint8_t* dst, size_t dst_capacity, bool single, size_t* consumed)
{
    int err = 0; uint64_t slot_bytes = 0;
    void* index = index_create(src, n, single, &slot_bytes, consumed, &err);
    if (!index) return err;
    FrameIndex& ix = *(FrameIndex*)index;
    int64_t rc = 0;
    uint8_t *d_src = nullptr, *d_slots = nullptr;
    cudaStream_t st = nullptr;
    std::vector<uint64_t> foff(ix.frames.size()), flen(ix.frames.size());
    std::vector<int32_t> blen(ix.blocks.size());
    do {
        if (b200lz4_device_count() <= 0) { rc = B200LZ4_E_NODEVICE; break; }
        if (cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking) != cudaSuccess ||
            cudaMalloc(&d_src, n + 16) != cudaSuccess || cudaMalloc(&d_slots, slot_bytes + 16) != cudaSuccess) { rc = B200LZ4_E_CUDA; break; }
        if (cudaMemcpyAsync(d_src, src, n, cudaMemcpyHostToDevice, st) != cudaSuccess) { rc = B200LZ4_E_CUDA; break; }
        rc = b200lz4f_decode_dev(index, d_src, d_slots, foff.data(), flen.data(), blen.data(), st);
        if (rc < 0 && rc != -11) break;
        // download: per frame when contiguous, else per run of blocks (short blocks in the middle of a frame)
        uint64_t pos = 0; bool ok = true;
        if (rc >= 0) {
            for (size_t f = 0; f < ix.frames.size() && ok; f++) {
                if (pos + flen[f] > dst_capacity) { rc = -9; ok = false; break; }
                if (flen[f] && cudaMemcpyAsync(dst + pos, d_slots + foff[f], flen[f], cudaMemcpyDeviceToHost, st) != cudaSuccess) { rc = B200LZ4_E_CUDA; ok = false; }
                pos += flen[f];
            }
        } else {
            // short blocks in mid-frame (everything is verified already): the device packs the blocks, one copy brings them back
            rc = 0;
            for (size_t b = 0; b < ix.blocks.size(); b++) pos += (uint64_t)blen[b];
            if (pos > dst_capacity) { rc = -9; ok = false; }
            uint8_t* d_tmp = nullptr;
            const size_t o_out = (pack_desc_bytes(ix.blocks.size()) + 15) & ~size_t(15);
            if (ok && pos) {
                if (cudaMalloc(&d_tmp, o_out + pos + 16) != cudaSuccess) { rc = B200LZ4_E_CUDA; ok = false; d_tmp = nullptr; }
                if (ok) {
                    if (pack_blocks(ix, blen.data(), d_slots, d_tmp + o_out, d_tmp, st) != cudaSuccess ||
                        cudaMemcpyAsync(dst, d_tmp + o_out, pos, cudaMemcpyDeviceToHost, st) != cudaSuccess ||
                        cudaStreamSynchronize(st) != cudaSuccess) { rc = B200LZ4_E_CUDA; ok = false; }
                }
            }
            if (d_tmp) cudaFree(d_tmp);
        }
        if (ok) { if (cudaStreamSynchronize(st) != cudaSuccess) rc = B200LZ4_E_CUDA; else rc = (int64_t)pos; }
    } while (0);
    if (d_src) cudaFree(d_src);
    if (d_slots) cudaFree(d_slots);
    if (st) cudaStreamDestroy(st);
    b200lz4f_index_free(index);
    return rc;
}

int64_t b200lz4f_decompress_host(const uint8_t* src, size_t n, uint8_t* dst, size_t dst_capacity)
{ return decompress_host(src, n, dst, dst_capacity, false, nullptr); }
// LZ4FrameInputStream(in, readSingleFrame = true): the first non-skippable frame only; *src_consumed = where it ended
int64_t b200lz4f_decompress_host_single(const uint8_t* src, size_t n, uint8_t* dst, size_t dst_capacity, size_t* src_consumed)
{ return decompress_host(src, n, dst, dst_capacity, true, src_consumed); }

// decompress_host with the container and the content in device memory: index on the device, decode into the thread's slot
// scratch, then one launch packs the blocks into d_dst.  Every verdict is in before the packing, so an error writes nothing.
int64_t b200lz4f_decompress_dev(const uint8_t* d_src, size_t n, uint8_t* d_dst, size_t dst_capacity, int single,
                                const uint64_t* frame_hint, size_t nhint, size_t* src_consumed, void* stream)
{
    if (!d_dst && dst_capacity) return fail_arg("null pointer");
    int err = 0; uint64_t slot_bytes = 0;
    void* index = b200lz4f_index_create_dev(d_src, n, single, frame_hint, nhint, &slot_bytes, src_consumed, &err, stream);
    if (!index) return err;
    const FrameIndex& ix = *(const FrameIndex*)index;
    const cudaStream_t st = (cudaStream_t)stream;
    std::vector<int32_t> blen(ix.blocks.size());
    FrameReadScratch* s;
    int64_t rc = get_frame_read_scratch(&s);
    if (!rc) rc = reserve_device(s->d_slots, s->slots_cap, slot_bytes + 16);
    if (!rc) rc = b200lz4f_decode_dev(index, d_src, s->d_slots, nullptr, nullptr, blen.data(), st);
    if (rc >= 0 || rc == -11) {
        uint64_t total = 0;
        for (const int32_t l : blen) total += (uint64_t)l;
        rc = total > dst_capacity ? -9 : reserve_device(s->d_pack, s->pack_cap, pack_desc_bytes(blen.size()));
        if (!rc) {
            cudaError_t e = pack_blocks(ix, blen.data(), s->d_slots, d_dst, s->d_pack, st);
            if (e == cudaSuccess) e = cudaStreamSynchronize(st);
            rc = e == cudaSuccess ? (int64_t)total : fail_cuda(e, "packing the decoded blocks");
        }
    }
    if (rc == B200LZ4_E_CUDA) cudaStreamSynchronize(st);
    b200lz4f_index_free(index);
    return rc;
}

} // extern "C"
