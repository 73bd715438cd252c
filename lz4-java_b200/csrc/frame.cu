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
#ifdef B200_HOST_SIM            // the emulator build compiles the host layer only: the device readers' kernels come with it
#include "frame_index.cu"
#include "frame_streams.cu"
#include "frame_reader.cu"
#endif
#include <algorithm>
#include <cstring>
#include <memory>
#include <new>
#include <vector>

namespace b200 {

struct FrameRec {
    uint64_t desc_off; int32_t desc_len; uint8_t hc_byte; uint8_t flg; uint32_t bs;
    uint64_t content_size; bool has_size;
    size_t first_block, nblocks;
    uint32_t content_checksum; bool has_checksum;
    uint64_t out_off;                   // slot-layout start of this frame's content
    bool complete;                      // read up to its EndMark (and content checksum); false: the container breaks off inside it
};

struct BlockRec { uint64_t src_off; uint32_t size; bool raw; uint32_t checksum; bool has_checksum; size_t frame; uint64_t out_off; uint32_t cap; };

// Where decode_dev's descriptor arrays lie in one blob of nb blocks (nc compressed, nr stored) and nf frames, nbsum block
// and nfsum content checksums; the same in the index, in d_seg and in h_seg.  The inputs come first and are uploaded, the
// results last: each of them comes back.
struct IndexLayout {
    size_t c_soff, c_doff, c_slen, c_dcap;                  // compressed blocks
    size_t r_soff, r_doff, r_len;                           // stored blocks
    size_t h_off, h_len, b_off, b_len;                      // what the descriptor and block checksums hash
    size_t f_first, f_nblk;                                 // content checksums (chained to the decoder: xxhash.cu)
    size_t k_comp, k_rawlen, k_off;                         // per block: index among the compressed blocks (-1: stored), stored size, slot
    size_t in, c_res, h_out, b_out, f_out, bytes = 0;       // in: the bytes of the inputs; then the results
    IndexLayout(size_t nb, size_t nc, size_t nr, size_t nf, size_t nbsum, size_t nfsum)
    {
        auto take = [&](size_t n) { const size_t at = bytes; bytes = (bytes + n + 15) & ~size_t(15); return at; };
        c_soff = take(8 * nc); c_doff = take(8 * nc); c_slen = take(4 * nc); c_dcap = take(4 * nc);
        r_soff = take(8 * nr); r_doff = take(8 * nr); r_len = take(4 * nr);
        h_off = take(8 * nf); h_len = take(4 * nf); b_off = take(8 * nbsum); b_len = take(4 * nbsum);
        f_first = take(4 * nfsum); f_nblk = take(4 * nfsum);
        k_comp = take(4 * nb); k_rawlen = take(4 * nb); k_off = take(8 * nb);
        in = bytes;
        c_res = take(4 * nc); h_out = take(4 * nf); b_out = take(4 * nbsum); f_out = take(4 * nfsum);
    }
};

// Host data only: nothing writes to an index once build_descriptors has run, so any number of threads may decode it at once.
struct FrameIndex {
    std::vector<FrameRec> frames;
    std::vector<BlockRec> blocks;
    uint64_t slot_bytes = 0;            // device bytes needed for the slot layout (upper bound of the decoded size)
    int tail_err = 0;                   // the container's own error, behind everything indexed (reported after what precedes it)
    size_t n_comp = 0, n_raw = 0, n_bsum = 0, n_fsum = 0;      // compressed and stored blocks, block and content checksums
    std::vector<uint8_t> blob;                                  // decode_dev's inputs, laid out by layout()
    IndexLayout layout() const { return IndexLayout(blocks.size(), n_comp, n_raw, frames.size(), n_bsum, n_fsum); }
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
        // the slot (frame_slot_room, kernels.h)
        const uint64_t room = frame_slot_room(f.bs, b.size, b.raw);
        b.cap = (uint32_t)room;
        b.out_off = ix.slot_bytes; ix.slot_bytes += frame_slot_bytes(room, f.bs);
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
        CK(cudaMemcpyAsync(D, s.h_seg, L.sums, cudaMemcpyHostToDevice, st));
        g_launch_count.fetch_add(3, std::memory_order_relaxed);
        CK(launch_frame_walk(d_src, n, single, (const WalkSeg*)D, (WalkSummary*)(D + L.sums), (int32_t*)(D + L.lens), (WalkRec*)s.d_recs, (uint32_t)k, st));
        CK(launch_scan((const int32_t*)(D + L.lens), (uint64_t*)(D + L.pos), (uint64_t*)(D + L.total), nullptr, k, st));
        CK(launch_frame_pack((const WalkSeg*)D, (const int32_t*)(D + L.lens), (const uint64_t*)(D + L.pos), (const WalkRec*)s.d_recs,
                             (WalkRec*)s.d_packed, (uint32_t)k, st));
        CK(cudaMemcpyAsync(s.h_seg + L.sums, D + L.sums, L.bytes - L.sums, cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        const uint64_t packed = *(const uint64_t*)(s.h_seg + L.total);
        const WalkSummary* hsum = (const WalkSummary*)(s.h_seg + L.sums);
        const uint64_t* hpos = (const uint64_t*)(s.h_seg + L.pos);
        std::vector<WalkSummary> got(hsum, hsum + k);
        std::vector<uint64_t> pos(hpos, hpos + k);
        if (packed) {
            CK(cudaMemcpyAsync(s.h_seg, s.d_packed, packed * sizeof(WalkRec), cudaMemcpyDeviceToHost, st));
            CK(cudaStreamSynchronize(st));
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
// The descriptors go up through d_seg / h_seg, free again once decode_dev has returned.  One launch; ordered on st.
static int pack_blocks(FrameReadScratch& s, const FrameIndex& ix, const int32_t* blen, const uint8_t* d_slots, uint8_t* d_dst, cudaStream_t st)
{
    const size_t nb = ix.blocks.size();
    if (nb == 0) return 0;
    const size_t o_to = (nb * 8 + 15) & ~size_t(15), o_len = 2 * o_to, bytes = o_len + nb * 4;
    int rc = reserve_device(s.d_seg, s.seg_cap, bytes);
    if (!rc) rc = reserve_pinned(s.h_seg, s.h_seg_cap, bytes);
    if (rc) return rc;
    uint8_t* h = s.h_seg;
    uint64_t pos = 0;
    for (size_t b = 0; b < nb; b++) {
        ((uint64_t*)h)[b] = ix.blocks[b].out_off;
        ((uint64_t*)(h + o_to))[b] = pos; pos += (uint64_t)blen[b];
    }
    memcpy(h + o_len, blen, nb * 4);
    CK(cudaMemcpyAsync(s.d_seg, h, bytes, cudaMemcpyHostToDevice, st));
    g_launch_count += 1;
    CK(launch_gather(d_slots, (const uint64_t*)s.d_seg, (const int32_t*)(s.d_seg + o_len), d_dst, (const uint64_t*)(s.d_seg + o_to), nb, st));
    return 0;
}

static int build_descriptors(FrameIndex& ix)
{
    for (const BlockRec& b : ix.blocks) { (b.raw ? ix.n_raw : ix.n_comp)++; ix.n_bsum += b.has_checksum; }
    for (const FrameRec& f : ix.frames) ix.n_fsum += f.has_checksum;
    const IndexLayout L = ix.layout();
    ix.blob.assign(L.in, 0);
    uint8_t* p = ix.blob.data();
    auto u64 = [&](size_t o) { return (uint64_t*)(p + o); };
    auto i32 = [&](size_t o) { return (int32_t*)(p + o); };
    size_t c = 0, r = 0, k = 0;
    for (size_t b = 0; b < ix.blocks.size(); b++) {
        const BlockRec& br = ix.blocks[b];
        u64(L.k_off)[b] = br.out_off;
        if (br.raw) {
            i32(L.k_comp)[b] = -1; i32(L.k_rawlen)[b] = (int32_t)br.size;
            u64(L.r_soff)[r] = br.src_off; u64(L.r_doff)[r] = br.out_off; i32(L.r_len)[r++] = (int32_t)br.size;
        } else {
            i32(L.k_comp)[b] = (int32_t)c;
            u64(L.c_soff)[c] = br.src_off; u64(L.c_doff)[c] = br.out_off; i32(L.c_slen)[c] = (int32_t)br.size; i32(L.c_dcap)[c++] = (int32_t)br.cap;
        }
        if (br.has_checksum) { u64(L.b_off)[k] = br.src_off; i32(L.b_len)[k++] = (int32_t)br.size; }
    }
    k = 0;
    for (size_t f = 0; f < ix.frames.size(); f++) {
        const FrameRec& fr = ix.frames[f];
        u64(L.h_off)[f] = fr.desc_off; i32(L.h_len)[f] = fr.desc_len;
        if (!fr.has_checksum) continue;
        if (fr.first_block > 0xFFFFFFFFull || fr.nblocks > 0xFFFFFFFFull) return -10;
        ((uint32_t*)(p + L.f_first))[k] = (uint32_t)fr.first_block; ((uint32_t*)(p + L.f_nblk))[k++] = (uint32_t)fr.nblocks;
    }
    return 0;
}

// ---- many independent frame streams in device memory (b200lz4f_decompress_streams_dev; kernels: frame_streams.cu)
// Where one call's per-stream arrays lie in d_seg / h_seg: the arguments and the zeroed `over` word go up; `over` and the
// scan totals come back after the counting walk, the results at the end.  The counts and their prefixes stay on the device.
struct FrameStreamLayout {
    size_t s_off, s_len, d_off, d_cap, over, totals, cnt, pos, tail, ip, result, consumed, content, bytes = 0;
    explicit FrameStreamLayout(size_t ns)
    {
        auto take = [&](size_t n) { const size_t at = bytes; bytes = (bytes + n + 15) & ~size_t(15); return at; };
        s_off = take(8 * ns); s_len = take(8 * ns); d_off = take(8 * ns); d_cap = take(8 * ns);
        over = take(4); totals = take(8 * FS_ROWS);
        cnt = take(4 * FS_ROWS * ns); pos = take(8 * FS_ROWS * ns); tail = take(4 * ns); ip = take(8 * ns);
        result = take(8 * ns); consumed = take(8 * ns); content = take(8 * ns);
    }
};
// ... and the records in d_recs, decode_dev's descriptor arrays for nc compressed and nr stored blocks, nbsum checksummed
// ones, nf frames and nfsum content checksums, with the verdict's per-frame facts and the packing's per-block destinations.
// They never leave the device.
struct FrameStreamRecLayout {
    size_t c_soff, c_doff, c_slen, c_dcap, c_res, r_soff, r_doff, r_len, k_comp, k_rawlen, k_off, k_dst, k_len;
    size_t b_off, b_len, b_want, b_out, h_off, h_len, h_out, fr_first, fr_nblk, fr_bsum, fr_fsum, fr_size, fr_bits;
    size_t f_first, f_nblk, f_want, f_out, bytes = 0;
    FrameStreamRecLayout(size_t nc, size_t nr, size_t nbsum, size_t nf, size_t nfsum)
    {
        auto take = [&](size_t n) { const size_t at = bytes; bytes = (bytes + n + 15) & ~size_t(15); return at; };
        const size_t nb = nc + nr;
        c_soff = take(8 * nc); c_doff = take(8 * nc); c_slen = take(4 * nc); c_dcap = take(4 * nc); c_res = take(4 * nc);
        r_soff = take(8 * nr); r_doff = take(8 * nr); r_len = take(4 * nr);
        k_comp = take(4 * nb); k_rawlen = take(4 * nb); k_off = take(8 * nb); k_dst = take(8 * nb); k_len = take(4 * nb);
        b_off = take(8 * nbsum); b_len = take(4 * nbsum); b_want = take(4 * nbsum); b_out = take(4 * nbsum);
        h_off = take(8 * nf); h_len = take(4 * nf); h_out = take(4 * nf);
        fr_first = take(4 * nf); fr_nblk = take(4 * nf); fr_bsum = take(4 * nf); fr_fsum = take(4 * nf); fr_size = take(8 * nf);
        fr_bits = take(4 * nf);
        f_first = take(4 * nfsum); f_nblk = take(4 * nfsum); f_want = take(4 * nfsum); f_out = take(4 * nfsum);
    }
};

// Points r's record arrays into the call's record region B.
static void bind_stream_records(FrameStreamRead& r, uint8_t* B, const FrameStreamRecLayout& R)
{
    r.c_soff = (uint64_t*)(B + R.c_soff); r.c_doff = (uint64_t*)(B + R.c_doff);
    r.c_slen = (int32_t*)(B + R.c_slen); r.c_dcap = (int32_t*)(B + R.c_dcap); r.c_res = (int32_t*)(B + R.c_res);
    r.r_soff = (uint64_t*)(B + R.r_soff); r.r_doff = (uint64_t*)(B + R.r_doff); r.r_len = (int32_t*)(B + R.r_len);
    r.k_comp = (int32_t*)(B + R.k_comp); r.k_rawlen = (int32_t*)(B + R.k_rawlen); r.k_off = (uint64_t*)(B + R.k_off);
    r.k_dst = (uint64_t*)(B + R.k_dst); r.k_len = (int32_t*)(B + R.k_len);
    r.b_off = (uint64_t*)(B + R.b_off); r.b_len = (int32_t*)(B + R.b_len); r.b_want = (uint32_t*)(B + R.b_want); r.b_out = (uint32_t*)(B + R.b_out);
    r.h_off = (uint64_t*)(B + R.h_off); r.h_len = (int32_t*)(B + R.h_len); r.h_out = (uint32_t*)(B + R.h_out);
    r.fr_first = (uint32_t*)(B + R.fr_first); r.fr_nblk = (uint32_t*)(B + R.fr_nblk); r.fr_bsum = (int32_t*)(B + R.fr_bsum);
    r.fr_fsum = (int32_t*)(B + R.fr_fsum); r.fr_size = (uint64_t*)(B + R.fr_size); r.fr_bits = (uint32_t*)(B + R.fr_bits);
    r.f_first = (uint32_t*)(B + R.f_first); r.f_nblk = (uint32_t*)(B + R.f_nblk); r.f_want = (uint32_t*)(B + R.f_want); r.f_out = (uint32_t*)(B + R.f_out);
}

// decode_dev's payload launches behind a recording walk: descriptor and block checksums, stored blocks, then every compressed
// block; the content checksums follow the decoder on the side stream (with carry / mode: launch_xxh32_frames_chained_carry).
static int stream_payload_launches(const FrameStreamRead& r, uint8_t* slots, uint64_t bytes, uint64_t nc, uint64_t nr,
                                   uint64_t nbsum, uint64_t nf, uint64_t nfsum, SideStream* side, cudaStream_t st,
                                   Xxh32Carry* carry = nullptr, const uint8_t* mode = nullptr)
{
    const uint64_t nb = nc + nr;
    if (nc) CK(cudaMemsetAsync(r.c_res, 0x80, nc * 4, st));                  // FRAME_RES_PENDING
    if (nf) CK(counted(launch_xxh32(r.src, r.h_off, r.h_len, 0, r.h_out, (size_t)nf, st)));
    if (nbsum)                      // the average stream byte per block bounds the average checksummed block
        CK(counted((bytes / nb >= XXH_LONG_AVG ? launch_xxh32_long : launch_xxh32)(r.src, r.b_off, r.b_len, 0, r.b_out, (size_t)nbsum, st)));
    if (nr) CK(counted(launch_gather(r.src, r.r_soff, r.r_len, slots, r.r_doff, (size_t)nr, st)));
    CK(cudaEventRecord(side->fork, st));
    if (nc) {
        const BatchArgs a{ r.src, r.c_soff, r.c_slen, slots, r.c_doff, r.c_dcap, r.c_res, (size_t)nc };
        CK(counted(launch_decompress_safe(a, st)));
    }
    if (nfsum) {
        CK(cudaStreamWaitEvent(side->st, side->fork, 0));
        if (carry)
            CK(counted(launch_xxh32_frames_chained_carry(slots, r.k_off, r.f_first, r.f_nblk, r.k_comp, r.k_rawlen, r.c_res, r.f_out,
                                                         (size_t)nfsum, carry, mode, side->st)));
        else
            CK(counted(launch_xxh32_frames_chained(slots, r.k_off, r.f_first, r.f_nblk, r.k_comp, r.k_rawlen, r.c_res, r.f_out,
                                                   (size_t)nfsum, side->st)));
        CK(cudaEventRecord(side->join, side->st));
        CK(cudaStreamWaitEvent(st, side->join, 0));
    }
    return 0;
}

// decode_dev for many streams at once with the index built and judged on the device: counting walk, scans of the counts (only
// their totals come to the host, to size the records and slots), recording walk, decode_dev's payload launches, one verdict
// warp per stream, one gather into d_dst.  The launches do not depend on the number of streams, frames or blocks.
static int frame_streams_decompress_dev(const uint8_t* d_src, const uint64_t* src_off, const uint64_t* src_len, size_t ns,
                                        uint8_t* d_dst, const uint64_t* dst_off, const uint64_t* dst_cap, bool single,
                                        int64_t* result, uint64_t* src_consumed, uint64_t* content_len, cudaStream_t st)
{
    if (ns == 0) return 0;
    if (!src_off || !src_len || !dst_off || !dst_cap || !result) return fail_arg("null pointer");
    if (ns > 0x7FFFFFFFull) return fail_arg("too many streams in one call");
    uint64_t bytes, room;
    int rc = check_stream_ranges(ns, src_len, 1ull << 47, dst_off, dst_cap, d_src, d_dst, bytes, room);
    if (rc) return rc;
    FrameReadScratch* s; SideStream* side;
    rc = get_frame_read_scratch(&s, &side);
    const FrameStreamLayout L(ns);
    if (!rc) rc = reserve_device(s->d_seg, s->seg_cap, L.bytes);
    if (!rc) rc = reserve_pinned(s->h_seg, s->h_seg_cap, L.bytes);
    if (rc) return rc;
    uint8_t *D = s->d_seg, *H = s->h_seg;
    memcpy(H + L.s_off, src_off, 8 * ns); memcpy(H + L.s_len, src_len, 8 * ns);
    memcpy(H + L.d_off, dst_off, 8 * ns); memcpy(H + L.d_cap, dst_cap, 8 * ns);
    memset(H + L.over, 0, 4);
    FrameStreamRead r{};
    r.src = d_src;
    r.s_off = (const uint64_t*)(D + L.s_off); r.s_len = (const uint64_t*)(D + L.s_len);
    r.d_off = (const uint64_t*)(D + L.d_off); r.d_cap = (const uint64_t*)(D + L.d_cap);
    r.cnt = (int32_t*)(D + L.cnt); r.pos = (const uint64_t*)(D + L.pos);
    r.tail = (int32_t*)(D + L.tail); r.ip = (uint64_t*)(D + L.ip); r.over = (int32_t*)(D + L.over);
    r.result = (int64_t*)(D + L.result); r.consumed = (uint64_t*)(D + L.consumed); r.content = (uint64_t*)(D + L.content);
    r.ns = (uint32_t)ns; r.single = single;
    uint64_t* totals = (uint64_t*)(D + L.totals);

    Drain drain{ st, side->st };
    CK(cudaMemcpyAsync(D, H, L.totals, cudaMemcpyHostToDevice, st));
    g_launch_count.fetch_add(1 + FS_ROWS, std::memory_order_relaxed);
    CK(launch_frame_streams_walk(r, false, st));
    for (int row = 0; row < FS_ROWS; row++)
        CK(launch_scan(r.cnt + row * ns, (uint64_t*)r.pos + row * ns, totals + row, nullptr, ns, st));
    CK(cudaMemcpyAsync(H + L.over, D + L.over, L.cnt - L.over, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    const uint64_t* tot = (const uint64_t*)(H + L.totals);
    const uint64_t nc = tot[FS_COMP], nr = tot[FS_RAW], nb = nc + nr, nbsum = tot[FS_BSUM], nf = tot[FS_FRAME], nfsum = tot[FS_FSUM];
    const uint64_t slot_bytes = tot[FS_SLOT16] << 4;
    if (*(const int32_t*)(H + L.over) || nb > 0x7FFFFFFFull || nf > 0x7FFFFFFFull)
        return fail_arg("more than 2^31 - 1 blocks or frames in one call, or 32 GiB of decode slots in one stream");
    const FrameStreamRecLayout R(nc, nr, nbsum, nf, nfsum);
    rc = reserve_device(s->d_recs, s->recs_cap, R.bytes + 16);
    if (!rc) rc = reserve_device(s->d_slots, s->slots_cap, slot_bytes + 16);
    if (rc) return rc;
    uint8_t* slots = s->d_slots;
    bind_stream_records(r, s->d_recs, R);

    CK(counted(launch_frame_streams_walk(r, true, st)));
    rc = stream_payload_launches(r, slots, bytes, nc, nr, nbsum, nf, nfsum, side, st);
    if (rc) return rc;
    // every verdict is in before anything is packed: a stream that fails writes nothing in d_dst
    CK(counted(launch_frame_streams_verdict(r, st)));
    if (nb) CK(counted(launch_gather(slots, r.k_off, r.k_len, d_dst, r.k_dst, (size_t)nb, st)));
    CK(cudaMemcpyAsync(H + L.result, D + L.result, L.bytes - L.result, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    drain.done = true;
    memcpy(result, H + L.result, 8 * ns);
    if (src_consumed) memcpy(src_consumed, H + L.consumed, 8 * ns);
    if (content_len) memcpy(content_len, H + L.content, 8 * ns);
    return 0;
}

// ---- the incremental reader (b200lz4f_reader_*; kernels: frame_reader.cu).  The reader is host data: one state per stream.
struct FrameReaderHandle {
    size_t ns; bool single;
    std::vector<FrameReaderState> st;
};
// One call's per-stream arrays in d_seg / h_seg: the arguments, the states and the zeroed `over` word go up; `over` and the
// scan totals come back after the counting walk, the results and the new states at the end.
struct FrameReaderLayout {
    size_t s_off, s_len, d_off, d_cap, eof, st_in, over, totals, cnt, pos, tail, status, consumed, produced, need, st_out, bytes = 0;
    explicit FrameReaderLayout(size_t ns)
    {
        auto take = [&](size_t n) { const size_t at = bytes; bytes = (bytes + n + 15) & ~size_t(15); return at; };
        s_off = take(8 * ns); s_len = take(8 * ns); d_off = take(8 * ns); d_cap = take(8 * ns); eof = take(ns);
        st_in = take(sizeof(FrameReaderState) * ns);
        over = take(4); totals = take(8 * FS_ROWS);
        cnt = take(4 * FS_ROWS * ns); pos = take(8 * FS_ROWS * ns); tail = take(4 * ns);
        status = take(4 * ns); consumed = take(8 * ns); produced = take(8 * ns); need = take(8 * ns);
        st_out = take(sizeof(FrameReaderState) * ns);
    }
};

// frame_streams_decompress_dev's steps from each stream's carried state: counting walk, scans (their totals come to the
// host), recording walk, decode_dev's payload launches with the carried content checksums, one verdict warp per stream,
// one gather of the blocks in front of each stream's cut.
static int frame_reader_read_dev(FrameReaderHandle* h, const uint8_t* d_src, const uint64_t* src_off, const uint64_t* src_len,
                                 const uint8_t* eof, uint8_t* d_dst, const uint64_t* dst_off, const uint64_t* dst_cap,
                                 int32_t* status, uint64_t* src_consumed, uint64_t* produced, uint64_t* need, cudaStream_t st)
{
    if (!h) return fail_arg("null reader");
    const size_t ns = h->ns;
    if (ns == 0) return 0;
    if (!src_off || !src_len || !eof || !dst_off || !dst_cap || !status || !src_consumed || !produced || !need)
        return fail_arg("null pointer");
    uint64_t bytes, room;
    int rc = check_stream_ranges(ns, src_len, 1ull << 47, dst_off, dst_cap, d_src, d_dst, bytes, room);
    if (rc) return rc;
    FrameReadScratch* s; SideStream* side;
    rc = get_frame_read_scratch(&s, &side);
    const FrameReaderLayout L(ns);
    if (!rc) rc = reserve_device(s->d_seg, s->seg_cap, L.bytes);
    if (!rc) rc = reserve_pinned(s->h_seg, s->h_seg_cap, L.bytes);
    if (rc) return rc;
    uint8_t *D = s->d_seg, *H = s->h_seg;
    memcpy(H + L.s_off, src_off, 8 * ns); memcpy(H + L.s_len, src_len, 8 * ns);
    memcpy(H + L.d_off, dst_off, 8 * ns); memcpy(H + L.d_cap, dst_cap, 8 * ns); memcpy(H + L.eof, eof, ns);
    memcpy(H + L.st_in, h->st.data(), sizeof(FrameReaderState) * ns);
    memset(H + L.over, 0, 4);
    FrameReaderRead q{};
    FrameStreamRead& r = q.r;
    r.src = d_src;
    r.s_off = (const uint64_t*)(D + L.s_off); r.s_len = (const uint64_t*)(D + L.s_len);
    r.d_off = (const uint64_t*)(D + L.d_off); r.d_cap = (const uint64_t*)(D + L.d_cap);
    r.cnt = (int32_t*)(D + L.cnt); r.pos = (const uint64_t*)(D + L.pos);
    r.tail = (int32_t*)(D + L.tail); r.over = (int32_t*)(D + L.over); r.consumed = (uint64_t*)(D + L.consumed);
    r.ns = (uint32_t)ns; r.single = h->single;
    q.eof = D + L.eof;
    q.st_in = (const FrameReaderState*)(D + L.st_in); q.st_out = (FrameReaderState*)(D + L.st_out);
    q.status = (int32_t*)(D + L.status); q.produced = (uint64_t*)(D + L.produced); q.need = (uint64_t*)(D + L.need);
    uint64_t* totals = (uint64_t*)(D + L.totals);

    Drain drain{ st, side->st };
    CK(cudaMemcpyAsync(D, H, L.totals, cudaMemcpyHostToDevice, st));
    g_launch_count.fetch_add(1 + FS_ROWS, std::memory_order_relaxed);
    CK(launch_frame_reader_walk(q, false, st));
    for (int row = 0; row < FS_ROWS; row++)
        CK(launch_scan(r.cnt + row * ns, (uint64_t*)r.pos + row * ns, totals + row, nullptr, ns, st));
    CK(cudaMemcpyAsync(H + L.over, D + L.over, L.cnt - L.over, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    const uint64_t* tot = (const uint64_t*)(H + L.totals);
    const uint64_t nc = tot[FS_COMP], nr = tot[FS_RAW], nb = nc + nr, nbsum = tot[FS_BSUM], nf = tot[FS_FRAME], nfsum = tot[FS_FSUM];
    const uint64_t slot_bytes = tot[FS_SLOT16] << 4;
    if (*(const int32_t*)(H + L.over) || nb > 0x7FFFFFFFull || nf > 0x7FFFFFFFull)
        return fail_arg("more than 2^31 - 1 blocks or frames in one call, or 32 GiB of decode slots in one stream");
    // decode_dev's records, then the reader's own: unit starts, frame parts, carried content checksums
    const FrameStreamRecLayout R(nc, nr, nbsum, nf, nfsum);
    size_t x = R.bytes;
    auto take = [&](size_t n) { const size_t at = x; x = (x + n + 15) & ~size_t(15); return at; };
    const size_t k_at = take(8 * nb), fr_at = take(8 * nf), fr_end_at = take(8 * nf), fr_mode = take(4 * nf);
    const size_t f_carry = take(sizeof(Xxh32Carry) * nfsum), f_mode = take(nfsum);
    rc = reserve_device(s->d_recs, s->recs_cap, x + 16);
    if (!rc) rc = reserve_device(s->d_slots, s->slots_cap, slot_bytes + 16);
    if (rc) return rc;
    uint8_t *B = s->d_recs, *slots = s->d_slots;
    bind_stream_records(r, B, R);
    q.k_at = (uint64_t*)(B + k_at); q.fr_at = (uint64_t*)(B + fr_at); q.fr_end_at = (uint64_t*)(B + fr_end_at);
    q.fr_mode = (uint32_t*)(B + fr_mode); q.f_carry = (Xxh32Carry*)(B + f_carry); q.f_mode = B + f_mode;

    CK(counted(launch_frame_reader_walk(q, true, st)));
    rc = stream_payload_launches(r, slots, bytes, nc, nr, nbsum, nf, nfsum, side, st, q.f_carry, q.f_mode);
    if (rc) return rc;
    CK(counted(launch_frame_reader_verdict(q, st)));
    if (nb) CK(counted(launch_gather(slots, r.k_off, r.k_len, d_dst, r.k_dst, (size_t)nb, st)));
    CK(cudaMemcpyAsync(H + L.status, D + L.status, L.bytes - L.status, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    drain.done = true;
    memcpy(status, H + L.status, 4 * ns);
    memcpy(src_consumed, H + L.consumed, 8 * ns);
    memcpy(produced, H + L.produced, 8 * ns);
    memcpy(need, H + L.need, 8 * ns);
    memcpy(h->st.data(), H + L.st_out, sizeof(FrameReaderState) * ns);
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

void b200lz4f_index_free(void* index) { delete (FrameIndex*)index; }

// Decode every indexed frame: d_src holds the container bytes, d_slots (>= slot_bytes) receives block b at its slot
// (b200lz4f_index_block_offsets; full blocks of one frame lie back to back).  On success frame_off[f] / frame_len[f] (host
// arrays, may be NULL) describe each frame's content, one run inside d_slots when no block was flushed short mid-frame;
// otherwise -11 is returned after every check has passed and the caller reads block by block (the host path below does).
// The descriptors go up from, and the results come back into, the thread's reader scratch: the index is only read.
// Returns total decoded bytes or a negative code.
int64_t b200lz4f_decode_dev(void* index, const uint8_t* d_src, uint8_t* d_slots, uint64_t* frame_off, uint64_t* frame_len,
                            int32_t* block_len_out, void* stream)
{
    const FrameIndex& ix = *(const FrameIndex*)index;
    const cudaStream_t st = (cudaStream_t)stream;
    const IndexLayout L = ix.layout();
    FrameReadScratch* s; SideStream* side;
    int rc = get_frame_read_scratch(&s, &side);
    if (!rc) rc = reserve_device(s->d_seg, s->seg_cap, L.bytes + 16);
    if (!rc) rc = reserve_pinned(s->h_seg, s->h_seg_cap, L.bytes);
    if (rc) return rc;
    uint8_t *D = s->d_seg, *H = s->h_seg;
    const size_t nf = ix.frames.size();
    std::copy(ix.blob.begin(), ix.blob.end(), H);
    Drain drain{ st, side->st };
    CK(cudaMemcpyAsync(D, H, L.in, cudaMemcpyHostToDevice, st));
    if (ix.n_comp) CK(cudaMemsetAsync(D + L.c_res, 0x80, ix.n_comp * 4, st));       // FRAME_RES_PENDING
    // 1. header + block checksums
    g_launch_count += 1;
    CK(launch_xxh32(d_src, (uint64_t*)(D + L.h_off), (int32_t*)(D + L.h_len), 0, (uint32_t*)(D + L.h_out), nf, st));
    if (ix.n_bsum) {
        // few long payloads: one warp per stream; many short ones: one lane per buffer (xxhash.cu)
        uint64_t sum = 0; for (const BlockRec& b : ix.blocks) if (b.has_checksum) sum += b.size;
        g_launch_count += 1;
        CK((sum / ix.n_bsum >= XXH_LONG_AVG ? launch_xxh32_long : launch_xxh32)(
               d_src, (uint64_t*)(D + L.b_off), (int32_t*)(D + L.b_len), 0, (uint32_t*)(D + L.b_out), ix.n_bsum, st));
    }
    // 2. stored blocks are copied, then every compressed block is decoded; 3. one warp per frame folds the blocks into the
    // content checksum as the decoder hands them over (side stream; the decode kernel is launched FIRST and waits for nobody)
    if (ix.n_raw) {
        g_launch_count += 1;
        CK(launch_gather(d_src, (uint64_t*)(D + L.r_soff), (int32_t*)(D + L.r_len), d_slots, (uint64_t*)(D + L.r_doff), ix.n_raw, st));
    }
    CK(cudaEventRecord(side->fork, st));
    if (ix.n_comp) {
        BatchArgs a{ d_src, (uint64_t*)(D + L.c_soff), (int32_t*)(D + L.c_slen), d_slots, (uint64_t*)(D + L.c_doff),
                     (int32_t*)(D + L.c_dcap), (int32_t*)(D + L.c_res), ix.n_comp };
        g_launch_count += 1;
        CK(launch_decompress_safe(a, st));
    }
    if (ix.n_fsum) {
        CK(cudaStreamWaitEvent(side->st, side->fork, 0));
        g_launch_count += 1;
        CK(launch_xxh32_frames_chained(d_slots, (uint64_t*)(D + L.k_off), (uint32_t*)(D + L.f_first), (uint32_t*)(D + L.f_nblk),
                                       (int32_t*)(D + L.k_comp), (int32_t*)(D + L.k_rawlen), (int32_t*)(D + L.c_res),
                                       (uint32_t*)(D + L.f_out), ix.n_fsum, side->st));
        CK(cudaEventRecord(side->join, side->st));
        CK(cudaStreamWaitEvent(st, side->join, 0));
    }
    if (ix.n_comp) CK(cudaMemcpyAsync(H + L.c_res, D + L.c_res, ix.n_comp * 4, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(H + L.h_out, D + L.h_out, nf * 4, cudaMemcpyDeviceToHost, st));
    if (ix.n_bsum) CK(cudaMemcpyAsync(H + L.b_out, D + L.b_out, ix.n_bsum * 4, cudaMemcpyDeviceToHost, st));
    if (ix.n_fsum) CK(cudaMemcpyAsync(H + L.f_out, D + L.f_out, ix.n_fsum * 4, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    drain.done = true;

    // the verdict, in the order the stream reader meets things: frame by frame -- descriptor hash (:208-216), then block by
    // block its checksum (:298-303) and its decode (:307-311), then at the EndMark content checksum (:266-269) and size
    // (:270-272).  Each kind of result is in block or frame order, so a running count finds the next one.
    const uint32_t *h_out = (const uint32_t*)(H + L.h_out), *b_out = (const uint32_t*)(H + L.b_out), *f_out = (const uint32_t*)(H + L.f_out);
    const int32_t* c_res = (const int32_t*)(H + L.c_res);
    size_t kc = 0, kb = 0, kf = 0;
    std::vector<int32_t> blen(ix.blocks.size());
    int64_t total = 0; bool gaps = false;
    for (size_t f = 0; f < nf; f++) {
        const FrameRec& fr = ix.frames[f];
        if (((h_out[f] >> 8) & 0xFF) != fr.hc_byte) return -3;
        uint64_t len = 0;
        for (size_t k = 0; k < fr.nblocks; k++) {
            const size_t b = fr.first_block + k;
            const BlockRec& br = ix.blocks[b];
            if (br.has_checksum && b_out[kb++] != br.checksum) return -5;
            int32_t l = (int32_t)br.size;
            if (!br.raw) { l = c_res[kc++]; if (l < 0) return -6; }              // LZ4Exception -> IOException
            blen[b] = l;
            if (k + 1 < fr.nblocks && (uint32_t)l != fr.bs) gaps = true;          // a short block in the middle of a frame
            len += (uint64_t)l;
        }
        if (fr.has_checksum && f_out[kf++] != fr.content_checksum) return -7;
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

// Whole thing with HOST buffers: index, upload, decode, download into one contiguous stream.  Runs on a stream of the thread's
// context.  The container, the slots and the packed content are device memory of this call only, freed before it returns.
static int64_t decompress_host(const uint8_t* src, size_t n, uint8_t* dst, size_t dst_capacity, bool single, size_t* consumed)
{
    int err = 0; uint64_t slot_bytes = 0;
    const std::unique_ptr<FrameIndex> ix((FrameIndex*)index_create(src, n, single, &slot_bytes, consumed, &err));
    if (!ix) return err;
    FrameReadScratch* s; cudaStream_t st;
    int rc = get_frame_read_scratch(&s, nullptr, &st);
    if (rc) return rc;
    struct CallBuffer { uint8_t* p = nullptr; ~CallBuffer() { if (p) cudaFree(p); } } d_src, d_slots, d_out;
    CK(cudaMalloc(&d_src.p, n + 16));
    CK(cudaMalloc(&d_slots.p, slot_bytes + 16));
    const size_t nf = ix->frames.size();
    std::vector<uint64_t> foff(nf), flen(nf);
    std::vector<int32_t> blen(ix->blocks.size());
    Drain drain{ st };
    CK(cudaMemcpyAsync(d_src.p, src, n, cudaMemcpyHostToDevice, st));
    const int64_t got = b200lz4f_decode_dev(ix.get(), d_src.p, d_slots.p, foff.data(), flen.data(), blen.data(), st);
    if (got < 0 && got != -11) return got;
    uint64_t total = 0;
    for (const int32_t l : blen) total += (uint64_t)l;
    if (total > dst_capacity) return -9;
    if (got >= 0) {                 // every frame is one run in the slots: one copy each
        for (size_t f = 0, pos = 0; f < nf; pos += flen[f++])
            if (flen[f]) CK(cudaMemcpyAsync(dst + pos, d_slots.p + foff[f], flen[f], cudaMemcpyDeviceToHost, st));
    } else if (total) {             // short blocks mid-frame: the device packs the blocks, one copy brings them back
        CK(cudaMalloc(&d_out.p, total + 16));
        rc = pack_blocks(*s, *ix, blen.data(), d_slots.p, d_out.p, st);
        if (rc) return rc;
        CK(cudaMemcpyAsync(dst, d_out.p, total, cudaMemcpyDeviceToHost, st));
    }
    CK(cudaStreamSynchronize(st));
    drain.done = true;
    return (int64_t)total;
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
    const std::unique_ptr<FrameIndex> ix((FrameIndex*)b200lz4f_index_create_dev(d_src, n, single, frame_hint, nhint, &slot_bytes,
                                                                                 src_consumed, &err, stream));
    if (!ix) return err;
    const cudaStream_t st = (cudaStream_t)stream;
    std::vector<int32_t> blen(ix->blocks.size());
    FrameReadScratch* s;
    int64_t rc = get_frame_read_scratch(&s);
    if (!rc) rc = reserve_device(s->d_slots, s->slots_cap, slot_bytes + 16);
    if (!rc) rc = b200lz4f_decode_dev(ix.get(), d_src, s->d_slots, nullptr, nullptr, blen.data(), st);
    if (rc < 0 && rc != -11) return rc;
    uint64_t total = 0;
    for (const int32_t l : blen) total += (uint64_t)l;
    if (total > dst_capacity) return -9;
    Drain drain{ st };
    rc = pack_blocks(*s, *ix, blen.data(), s->d_slots, d_dst, st);
    if (rc) return rc;
    CK(cudaStreamSynchronize(st));
    drain.done = true;
    return (int64_t)total;
}

// ns frame streams, each read like b200lz4f_decompress_host{,_single} would read it alone (frame_streams_decompress_dev)
int b200lz4f_decompress_streams_dev(const uint8_t* d_src, const uint64_t* src_off, const uint64_t* src_len, size_t ns,
                                    uint8_t* d_dst, const uint64_t* dst_off, const uint64_t* dst_cap, int single,
                                    int64_t* result, uint64_t* src_consumed, uint64_t* content_len, void* stream)
{
    return frame_streams_decompress_dev(d_src, src_off, src_len, ns, d_dst, dst_off, dst_cap, single != 0, result, src_consumed,
                                        content_len, (cudaStream_t)stream);
}

// the incremental reader (frame_reader_read_dev): host data only, no CUDA call in create or free
void* b200lz4f_reader_create(size_t ns, int single, int* err)
{
    if (err) *err = 0;
    if (ns > 0x7FFFFFFFull) { const int rc = fail_arg("too many streams in one reader"); if (err) *err = rc; return nullptr; }
    FrameReaderHandle* h = new (std::nothrow) FrameReaderHandle;
    if (!h) { const int rc = fail_arg("out of host memory"); if (err) *err = rc; return nullptr; }
    h->ns = ns; h->single = single != 0;
    try { h->st.assign(ns, FrameReaderState{}); }
    catch (...) { delete h; const int rc = fail_arg("out of host memory"); if (err) *err = rc; return nullptr; }
    return h;
}

int b200lz4f_reader_read_dev(void* reader, const uint8_t* d_src, const uint64_t* src_off, const uint64_t* src_len,
                             const uint8_t* eof, uint8_t* d_dst, const uint64_t* dst_off, const uint64_t* dst_cap,
                             int32_t* status, uint64_t* src_consumed, uint64_t* produced, uint64_t* need, void* stream)
{
    return frame_reader_read_dev((FrameReaderHandle*)reader, d_src, src_off, src_len, eof, d_dst, dst_off, dst_cap, status,
                                 src_consumed, produced, need, (cudaStream_t)stream);
}

void b200lz4f_reader_free(void* reader) { delete (FrameReaderHandle*)reader; }

} // extern "C"
