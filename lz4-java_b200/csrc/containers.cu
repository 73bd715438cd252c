// containers.cu — the containers lz4-java wraps around the block codec, as whole-buffer batch calls:
//   * LZ4 Frame writer     — LZ4FrameOutputStream.writeHeader/writeBlock/writeEndMark
//                            (src/java/net/jpountz/lz4/LZ4FrameOutputStream.java:178-251)
//   * "LZ4Block" container — LZ4BlockOutputStream.flushBufferedData/finish (:203-266) and
//                            LZ4BlockInputStream.refill (LZ4BlockInputStream.java:191-264)
//   * length-prefixed block — LZ4CompressorWithLength / LZ4DecompressorWithLength
// The reference does these one block per native call.  Here all three containers are written on the device, by one loop
// (compress_blocks_dev) with the kernels of frame_encode.cu, lz4block.cu and with_length.cu; the host writers run it on a
// device copy of their source.  The LZ4Block reader walks the headers with walk_lz4block (kernels.h): on the host for host
// buffers, whose payload work (block decompression, every XXH32) goes through the batch entry points, and on the device for
// streams in device memory (lz4block.cu).  Length-prefixed records in device memory are read by with_length.cu's kernels
// around the block decoders.  No hashing or codec arithmetic runs on the host.
#include "../../include/b200lz4.h"
#include "kernels.h"
#ifdef B200_HOST_SIM            // the emulator build compiles the host layer only: the device writers' and readers' kernels come with it
#include "frame_encode.cu"
#include "frame_writer.cu"
#include "lz4block.cu"
#include "with_length.cu"
#endif
#include <cstdlib>
#include <cstring>
#include <vector>

static inline void put32(uint8_t* p, uint32_t v) { p[0] = (uint8_t)v; p[1] = (uint8_t)(v >> 8); p[2] = (uint8_t)(v >> 16); p[3] = (uint8_t)(v >> 24); }
static inline uint32_t get32(const uint8_t* p) { return p[0] | (p[1] << 8) | (p[2] << 16) | ((uint32_t)p[3] << 24); }

// ---------------------------------------------------------------- LZ4 Frame and LZ4Block writers (frame_encode.cu, lz4block.cu)
namespace b200 {

// Where the FramePlan arrays of a call with nb blocks, ni items and nf frames lie in one blob, the same on the host and the
// device.  f_off, f_end and the two carry words come last: one copy brings the results back.
// The incremental writer (nw = nf) adds per frame where its stream's range starts, its first item, its WRITER_* mode and its
// declared content size, and (nx = nf with a content checksum) the carried checksum's mode and state, which comes back too;
// the other writers have none of these (nw = nx = 0), and their layout is the same without them.
struct FramePlanLayout {
    size_t b_soff, b_slen, b_slot, b_ccap, b_clen, b_poff, b_plen, b_sum;
    size_t i_frame, i_block, i_size, i_off;
    size_t f_soff, f_len, f_len32, f_sum, f_doff, f_first, f_mode, f_known, f_xmode, f_off, f_end, f_xxh, carry, bytes = 0;
    FramePlanLayout(size_t nb, size_t ni, size_t nf, size_t nw = 0, size_t nx = 0)
    {
        auto take = [&](size_t n) { const size_t at = bytes; bytes = (bytes + n + 15) & ~size_t(15); return at; };
        b_soff = take(8 * nb); b_slen = take(4 * nb); b_slot = take(8 * nb); b_ccap = take(4 * nb); b_clen = take(4 * nb);
        b_poff = take(8 * nb); b_plen = take(4 * nb); b_sum = take(4 * nb);
        i_frame = take(4 * ni); i_block = take(4 * ni); i_size = take(4 * ni); i_off = take(8 * ni);
        f_soff = take(8 * nf); f_len = take(8 * nf); f_len32 = take(4 * nf); f_sum = take(4 * nf);
        f_doff = take(8 * nw); f_first = take(4 * nw); f_mode = take(nw); f_known = take(8 * nw); f_xmode = take(nx);
        f_off = take(8 * nf); f_end = take(8 * nf); f_xxh = take(sizeof(Xxh32Carry) * nx); carry = take(16);
    }
};

// items [i0, i1), their blocks [b0, b1): the fast compressor's wide kernel takes [b0, bw), its long kernel [bw, b1)
struct FrameChunk { size_t i0, i1, b0, b1, bw; };

// The three containers written on the device.  An LZ4Block "frame" is one stream: blocks of blockSize bytes, the end block on
// its last item, checksums of the original blocks.  A WithLength "frame" is one record: one item and one block of its whole
// length, an empty record included.
enum class Container { Frame, LZ4Block, WithLength };

static constexpr uint64_t LZ4_MAX_INPUT = 0x7E000000;              // LZ4_MAX_INPUT_SIZE (lz4.h:211)

// The plan of a writer call, into the pinned blob H laid out by L: frame f is src_len[f] bytes at src_off[f], cut into blocks
// of bs bytes (the last one short; a record is one block), one item per block or one item for an empty frame, and chunks of
// at most CHUNK_SPAN source bytes and CHUNK_BLOCKS items, so the compressed slots take the same room however large the call.
// Returns the slot room the largest chunk takes.
static uint64_t plan_blocks(Container kind, const FramePlanLayout& L, uint8_t* H, const uint64_t* src_off, const uint64_t* src_len,
                            size_t nf, uint64_t bs, std::vector<FrameChunk>& chunks)
{
    const bool rec = kind == Container::WithLength;
    auto h64 = [&](size_t o) { return (uint64_t*)(H + o); };
    auto h32 = [&](size_t o) { return (int32_t*)(H + o); };
    size_t b = 0, i = 0, ci0 = 0, cb0 = 0;
    uint64_t slot = 0, span = 0, slots_need = 0;
    // A chunk's blocks go to the wide compressor when they are at most 64 KiB (as b200lz4_compress_default picks it), else to
    // the long one.  Frame and LZ4Block blocks are all of one class.  Records are of either: the records of up to 64 KiB are
    // moved to the front of the chunk's blocks, so each class is one contiguous range and one launch; the items, and so the
    // scan and the output, stay in record order.
    auto close_chunk = [&](size_t i1) {
        size_t bw = bs <= 65536 ? b : cb0;
        if (rec) {
            struct Row { uint64_t soff, slot; int32_t slen, ccap; };
            std::vector<Row> rows(b - cb0);                             // block cb0 + k is item ci0 + k's
            for (size_t k = 0; k < rows.size(); k++)
                rows[k] = Row{ h64(L.b_soff)[cb0 + k], h64(L.b_slot)[cb0 + k], h32(L.b_slen)[cb0 + k], h32(L.b_ccap)[cb0 + k] };
            size_t w = cb0;
            for (int wide = 1; wide >= 0; wide--) {
                for (size_t k = 0; k < rows.size(); k++) {
                    if ((rows[k].slen <= 65536) != (wide == 1)) continue;
                    h64(L.b_soff)[w] = rows[k].soff; h64(L.b_slot)[w] = rows[k].slot;
                    h32(L.b_slen)[w] = rows[k].slen; h32(L.b_ccap)[w] = rows[k].ccap;
                    h32(L.i_block)[ci0 + k] = (int32_t)w; w++;
                }
                if (wide) bw = w;
            }
        }
        chunks.push_back(FrameChunk{ ci0, i1, cb0, b, bw });
    };
    for (size_t f = 0; f < nf; f++) {
        const uint64_t n = src_len[f], nbf = rec ? 1 : (n + bs - 1) / bs;
        h64(L.f_soff)[f] = src_off[f]; h64(L.f_len)[f] = n; h32(L.f_len32)[f] = (int32_t)(n < 0x7FFFFFFFull ? n : 0x7FFFFFFFull);
        for (uint64_t k = 0; k < (nbf ? nbf : 1); k++, i++) {
            const uint64_t len = nbf ? (n - k * bs < bs ? n - k * bs : bs) : 0;
            if (i > ci0 && (i - ci0 >= CHUNK_BLOCKS || span + len > CHUNK_SPAN)) {
                close_chunk(i);
                slots_need = slot > slots_need ? slot : slots_need;
                ci0 = i; cb0 = b; slot = 0; span = 0;
            }
            h32(L.i_frame)[i] = (int32_t)f;
            h32(L.i_block)[i] = nbf ? (int32_t)b : -1;
            if (!nbf) continue;
            h64(L.b_soff)[b] = src_off[f] + k * bs; h32(L.b_slen)[b] = (int32_t)len;
            h64(L.b_slot)[b] = slot; h32(L.b_ccap)[b] = (int32_t)compress_bound(len);
            slot += aligned_compress_bound(len); span += len; b++;
        }
    }
    close_chunk(i);
    h64(L.carry)[0] = 0;
    return slot > slots_need ? slot : slots_need;
}

// The chunk loop of every writer, ordered on st: per chunk the blocks are compressed into their slots, then the container's
// item sizes (sizes(i0, n)), the scan that places the items (the running offset carried from chunk to chunk in carry[0..1])
// and the container's emit (emit(i0, n)).  b_ccap: the blocks' slot capacities.
template <class Sizes, class Emit>
static int chunk_loop(const FramePlan& P, const int32_t* b_ccap, uint8_t* slots, const std::vector<FrameChunk>& chunks, int hc_level,
                      uint64_t* carry, Sizes sizes, Emit emit, cudaStream_t st)
{
    auto blocks = [&](size_t b0, size_t b1) {
        return BatchArgs{ P.src, P.b_soff + b0, P.b_slen + b0, slots, P.b_slot + b0, b_ccap + b0, (int32_t*)P.b_clen + b0, b1 - b0 };
    };
    for (size_t k = 0; k < chunks.size(); k++) {
        const FrameChunk& c = chunks[k];
        // the stream's compressor argument: hc_level 0 = the fast compressor, 1..17 = HC
        if (hc_level > 0 && c.b1 > c.b0) CK(counted(launch_compress_hc(blocks(c.b0, c.b1), hc_level, st)));
        if (hc_level <= 0 && c.bw > c.b0) CK(counted(launch_compress_fast(blocks(c.b0, c.bw), 65536, st)));
        if (hc_level <= 0 && c.b1 > c.bw) CK(counted(launch_compress_fast(blocks(c.bw, c.b1), 0, st)));
        const uint32_t i0 = (uint32_t)c.i0, n = (uint32_t)(c.i1 - c.i0);
        CK(counted(sizes(i0, n)));
        CK(counted(launch_scan(P.i_size + i0, P.i_off + i0, carry + ((k + 1) & 1), carry + (k & 1), n, st)));
        CK(counted(emit(i0, n)));
    }
    return 0;
}

// Every writer: arguments and sizes (nothing is launched or written before these pass), the plan, the chunk loop and the
// results.  Only the item sizes, the emit, the checksums and the seal differ by container.  bs: bytes per block (WithLength:
// more than any record); code: the frame's bsCode or the LZ4Block token's level nibble; flags: the frame's (0 otherwise).
static int64_t compress_blocks_dev(Container kind, const uint8_t* d_src, const uint64_t* src_off, const uint64_t* src_len,
                                   size_t nf, uint8_t* d_dst, size_t dst_capacity, uint64_t* frame_off, uint64_t* frame_len,
                                   uint64_t bs, int code, int flags, int hc_level, cudaStream_t st)
{
    const bool frame = kind == Container::Frame, rec = kind == Container::WithLength;
    if (nf == 0) return 0;
    if (!src_off || !src_len || !d_dst) return fail_arg("null pointer");
    uint64_t need = 0, nb = 0, ni = 0, bytes = 0;
    bool too_long = false;
    for (size_t f = 0; f < nf; f++) {
        const uint64_t n = src_len[f];
        if (n > (1ull << 47)) return fail_arg("src_len");
        if (rec && n > LZ4_MAX_INPUT) return fail_arg("a record is at most 0x7E000000 bytes");
        const uint64_t nbf = rec ? 1 : (n + bs - 1) / bs;
        need += frame ? b200lz4f_compress_bound(n, code) : rec ? 4 + compress_bound(n) : b200lz4block_compress_bound(n, (int)bs);
        nb += nbf; ni += nbf ? nbf : 1; bytes += n;
        if ((flags & 1) && n > 0x7FFFFFFFull) too_long = true;
    }
    if (bytes && !d_src) return fail_arg("null pointer");
    if (ni > 0x7FFFFFFFull) return fail_arg("too many blocks in one call");
    if (need > dst_capacity) return -9;
    if (too_long) return -10;                                       // the content checksum kernel takes 31-bit lengths (f_len32)
    FrameScratch* s; SideStream* side; int rc = get_frame_scratch(&s, &side); if (rc) return rc;
    const FramePlanLayout L(nb, ni, nf);
    rc = reserve_pinned(s->h_plan, s->h_plan_cap, L.bytes);
    if (!rc) rc = reserve_device(s->d_plan, s->plan_cap, L.bytes);
    if (rc) return rc;

    uint8_t* H = s->h_plan;
    auto h64 = [&](size_t o) { return (uint64_t*)(H + o); };
    std::vector<FrameChunk> chunks;
    const uint64_t slots_need = plan_blocks(kind, L, H, src_off, src_len, nf, bs, chunks);
    rc = reserve_device(s->d_slots, s->slots_cap, (size_t)slots_need + 16); if (rc) return rc;

    uint8_t* D = s->d_plan;
    const FramePlan P{ d_src, d_dst, s->d_slots,
                       (const uint64_t*)(D + L.b_soff), (const int32_t*)(D + L.b_slen), (const uint64_t*)(D + L.b_slot), (const int32_t*)(D + L.b_clen),
                       (uint64_t*)(D + L.b_poff), (int32_t*)(D + L.b_plen), (const uint32_t*)(D + L.b_sum),
                       (const uint32_t*)(D + L.i_frame), (const int32_t*)(D + L.i_block), (int32_t*)(D + L.i_size), (uint64_t*)(D + L.i_off),
                       (const uint64_t*)(D + L.f_len), (const uint32_t*)(D + L.f_sum), (uint64_t*)(D + L.f_off), (uint64_t*)(D + L.f_end),
                       (uint32_t)ni, frame ? code : 0, flags, frame ? 0 : code };
    uint64_t* carry = (uint64_t*)(D + L.carry);

    // ---- launches, all ordered after what `st` already holds
    Drain drain{ st, side->st };
    CK(cudaMemcpyAsync(D, H, L.bytes, cudaMemcpyHostToDevice, st));
    // checksums of the sources alone, so from the start, beside everything else: the frame's content checksums, or the
    // LZ4Block checksums of the original blocks (records have none)
    const bool early_sums = frame ? (flags & 1) != 0 : !rec && nb > 0;
    if (early_sums) {
        CK(cudaEventRecord(side->fork, st));
        CK(cudaStreamWaitEvent(side->st, side->fork, 0));
        if (frame)
            CK(counted(launch_xxh32_long(d_src, (const uint64_t*)(D + L.f_soff), (const int32_t*)(D + L.f_len32), 0,
                                         (uint32_t*)(D + L.f_sum), nf, side->st)));
        else
            CK(counted((bytes / nb >= XXH_LONG_AVG ? launch_xxh32_long : launch_xxh32)(
                d_src, P.b_soff, P.b_slen, LZ4BLOCK_SEED, (uint32_t*)P.b_sum, (size_t)nb, side->st)));
        CK(cudaEventRecord(side->join, side->st));
    }
    rc = chunk_loop(P, (const int32_t*)(D + L.b_ccap), s->d_slots, chunks, hc_level, carry,
                    [&](uint32_t i0, uint32_t n) { return frame ? launch_frame_sizes(P, i0, n, st) : rec ? launch_with_length_sizes(P, i0, n, st)
                                                                                                         : launch_lz4block_sizes(P, i0, n, st); },
                    [&](uint32_t i0, uint32_t n) { return frame ? launch_frame_emit(P, i0, n, st) : rec ? launch_with_length_emit(P, i0, n, st)
                                                                                                        : launch_lz4block_emit(P, i0, n, st); }, st);
    if (rc) return rc;
    if ((flags & 2) && nb) {        // block checksums over the payloads as written; the source average bounds the payloads'
        CK(counted((bytes / nb >= XXH_LONG_AVG ? launch_xxh32_long : launch_xxh32)(
            d_dst, P.b_poff, P.b_plen, 0, (uint32_t*)P.b_sum, (size_t)nb, st)));
    }
    if (early_sums) CK(cudaStreamWaitEvent(st, side->join, 0));
    if (!rec) CK(counted(frame ? launch_frame_seal(P, st) : launch_lz4block_seal(P, st)));   // records: the emit placed them
    CK(cudaMemcpyAsync(H + L.f_off, D + L.f_off, L.bytes - L.f_off, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    drain.done = true;
    for (size_t f = 0; f < nf; f++) {
        if (frame_off) frame_off[f] = h64(L.f_off)[f];
        if (frame_len) frame_len[f] = h64(L.f_end)[f] - h64(L.f_off)[f];
    }
    return (int64_t)h64(L.carry)[chunks.size() & 1];
}

static int64_t compress_frames_dev(const uint8_t* d_src, const uint64_t* src_off, const uint64_t* src_len, size_t nf,
                                   uint8_t* d_dst, size_t dst_capacity, uint64_t* frame_off, uint64_t* frame_len,
                                   int bsCode, int flags, int hc_level, cudaStream_t st)
{
    if (bsCode < 4 || bsCode > 7) return fail_arg("bsCode must be 4..7");
    return compress_blocks_dev(Container::Frame, d_src, src_off, src_len, nf, d_dst, dst_capacity, frame_off, frame_len,
                               1ull << (8 + 2 * bsCode), bsCode, flags, hc_level, st);
}

static int lz4block_level(int blockSize)                                        // LZ4BlockOutputStream.java:58-70
{
    int lvl = 0; while ((1 << lvl) < blockSize) lvl++;                           // 32 - numberOfLeadingZeros(blockSize - 1)
    lvl -= 10; return lvl < 0 ? 0 : lvl;
}

static int64_t compress_lz4block_dev(const uint8_t* d_src, const uint64_t* src_off, const uint64_t* src_len, size_t ns,
                                     uint8_t* d_dst, size_t dst_capacity, uint64_t* stream_off, uint64_t* stream_len,
                                     int blockSize, int hc_level, cudaStream_t st)
{
    if (blockSize < 64 || blockSize > (1 << 25)) return fail_arg("blockSize must be 64..32 MiB");
    return compress_blocks_dev(Container::LZ4Block, d_src, src_off, src_len, ns, d_dst, dst_capacity, stream_off, stream_len,
                               (uint64_t)blockSize, lz4block_level(blockSize), 0, hc_level, st);
}

static int64_t compress_with_length_dev(const uint8_t* d_src, const uint64_t* src_off, const uint64_t* src_len, size_t n,
                                        uint8_t* d_dst, size_t dst_capacity, uint64_t* rec_off, uint64_t* rec_len, int hc_level,
                                        cudaStream_t st)
{   // one block per record: bs is longer than any record may be
    return compress_blocks_dev(Container::WithLength, d_src, src_off, src_len, n, d_dst, dst_capacity, rec_off, rec_len,
                               1ull << 31, 0, 0, hc_level, st);
}

// ---- the incremental writers (b200lz4f_writer_*, b200lz4block_writer_*; kernels: frame_writer.cu, lz4block.cu).  A writer
// is host data: the streams' declared content sizes (frames with flags bit 2) and one state each.  bs: bytes per block; code:
// the frame's bsCode or the LZ4Block token's level nibble; flags: the frame's (0 for LZ4Block).
struct WriterHandle {
    Container kind; size_t ns; uint64_t bs; int code, flags, hc_level;
    std::vector<uint64_t> known;
    std::vector<FrameWriterState> st;
};

// A writer of ns streams with nothing written yet, or NULL when host memory runs out.  known: NULL, or ns declared sizes.
static WriterHandle* new_writer(Container kind, size_t ns, uint64_t bs, int code, int flags, int hc_level, const int64_t* known)
{
    WriterHandle* h = new (std::nothrow) WriterHandle{ kind, ns, bs, code, flags, hc_level };
    if (!h) return nullptr;
    try {
        if (known) h->known.assign((const uint64_t*)known, (const uint64_t*)known + ns);
        FrameWriterState w{};                       // XXH32 with seed 0, nothing hashed yet (xxhash.c:445-455)
        w.xxh.v[0] = 2654435761u + 2246822519u; w.xxh.v[1] = 2246822519u; w.xxh.v[2] = 0; w.xxh.v[3] = 0u - 2654435761u;
        h->st.assign(ns, w);
    } catch (...) { delete h; return nullptr; }
    return h;
}

// What a call does for one stream of an incremental writer, planned on the host from its piece's length, its op, its room
// and its state alone: the header if it is due and fits, then whole blocks while their bounds fit, the short tail at
// FLUSH / CLOSE, the stream's end at CLOSE.  The container's units: head the header's bytes (0: none due), word a block's
// bytes besides its payload, tail the end's bytes -- a frame's header, block word (and checksum) and EndMark (and content
// checksum); an LZ4Block stream's 21-byte block header and end block.  mode: WRITER_* for the plan.
struct WriterTake { uint64_t taken, need; int32_t status; uint8_t mode; };
struct WriterUnits { uint64_t head, word, tail; };
static WriterTake writer_take(bool done, uint64_t n, uint8_t op, uint64_t room, uint64_t bs, const WriterUnits& u)
{
    if (done) return { 0, 0, B200LZ4F_DONE, 0 };
    const uint64_t head = u.head, tail = u.tail, word = u.word;
    WriterTake t{ 0, 0, B200LZ4F_MORE_ROOM, 0 };
    if (head) {                                                         // writeHeader (:178-191)
        if (room < head) { t.need = head; return t; }
        room -= head; t.mode |= WRITER_HEAD;
    }
    const uint64_t whole = n / bs, fit = room / (bs + word), k = whole < fit ? whole : fit;
    t.taken = k * bs; room -= k * (bs + word);
    if (k < whole) { t.need = bs + word; return t; }
    const uint64_t rest = n - t.taken;
    if (op != B200LZ4F_WRITE && rest) {                                 // flush(): the rest as a short block (:199-241)
        if (room < rest + word) { t.need = rest + word; return t; }
        t.taken = n; room -= rest + word;
    }
    if (op == B200LZ4F_CLOSE) {                                         // close(): writeEndMark (:243-249)
        if (room < tail) { t.need = tail; return t; }
        t.mode |= WRITER_TAIL; t.status = B200LZ4F_DONE; return t;
    }
    t.status = B200LZ4F_MORE_INPUT; t.need = op == B200LZ4F_WRITE ? bs - rest : bs;
    return t;
}

// compress_blocks_dev's plan and chunk loop over the streams that write something, with the container's writer kernels: the
// plan up, the early checksums on the side stream from the start (a frame's carried content checksums, or LZ4Block's checksums
// of the original blocks), the chunks, the block checksums, the seal, each stream's range and checksum state back, one
// synchronisation.
static int writer_write_dev(WriterHandle* h, const uint8_t* d_src, const uint64_t* src_off, const uint64_t* src_len,
                            const uint8_t* op, uint8_t* d_dst, const uint64_t* dst_off, const uint64_t* dst_cap,
                            int32_t* status, uint64_t* src_consumed, uint64_t* produced, uint64_t* need, cudaStream_t st)
{
    if (!h) return fail_arg("null writer");
    const size_t ns = h->ns;
    if (ns == 0) return 0;
    if (!src_off || !src_len || !op || !dst_off || !dst_cap || !status || !src_consumed || !produced || !need)
        return fail_arg("null pointer");
    uint64_t bytes, room;
    int rc = check_stream_ranges(ns, src_len, 1ull << 47, dst_off, dst_cap, d_src, d_dst, bytes, room);
    if (rc) return rc;
    for (size_t k = 0; k < ns; k++)
        if (op[k] > B200LZ4F_CLOSE) return fail_arg("op must be B200LZ4F_WRITE, _FLUSH or _CLOSE");
    const bool frame = h->kind == Container::Frame;
    const int flags = h->flags;
    const uint64_t bs = h->bs;
    std::vector<WriterTake> take(ns);
    std::vector<uint64_t> p_soff, p_len;
    std::vector<uint32_t> p_stream;
    uint64_t nb = 0, ni = 0, taken = 0;
    for (size_t k = 0; k < ns; k++) {
        const WriterUnits u = frame ? WriterUnits{ h->st[k].head ? 0u : 7u + ((flags & 4) ? 8u : 0u), 4u + ((flags & 2) ? 4u : 0u),
                                                   4u + ((flags & 1) ? 4u : 0u) }
                                    : WriterUnits{ 0, LZ4BLOCK_HEADER, LZ4BLOCK_HEADER };
        take[k] = writer_take(h->st[k].done, src_len[k], op[k], dst_cap[k], bs, u);
        if (!take[k].mode && !take[k].taken) continue;
        const uint64_t nbf = (take[k].taken + bs - 1) / bs;
        p_soff.push_back(src_off[k]); p_len.push_back(take[k].taken); p_stream.push_back((uint32_t)k);
        nb += nbf; ni += nbf ? nbf : 1; taken += take[k].taken;
    }
    if (ni > 0x7FFFFFFFull) return fail_arg("more than 2^31 - 1 blocks in one call");
    const size_t nf = p_stream.size(), nx = (flags & 1) ? nf : 0;
    std::vector<uint64_t> range(ns, 0);
    std::vector<Xxh32Carry> xxh;
    if (nf) {
        FrameScratch* s; SideStream* side; rc = get_frame_scratch(&s, &side); if (rc) return rc;
        const FramePlanLayout L(nb, ni, nf, nf, nx);
        rc = reserve_pinned(s->h_plan, s->h_plan_cap, L.bytes);
        if (!rc) rc = reserve_device(s->d_plan, s->plan_cap, L.bytes);
        if (rc) return rc;
        uint8_t *H = s->h_plan, *D = s->d_plan;
        std::vector<FrameChunk> chunks;
        const uint64_t slots_need = plan_blocks(h->kind, L, H, p_soff.data(), p_len.data(), nf, bs, chunks);
        rc = reserve_device(s->d_slots, s->slots_cap, (size_t)slots_need + 16); if (rc) return rc;
        for (size_t f = 0, i = 0; f < nf; f++) {
            const size_t k = p_stream[f];
            ((uint64_t*)(H + L.f_doff))[f] = dst_off[k];
            ((uint32_t*)(H + L.f_first))[f] = (uint32_t)i;
            (H + L.f_mode)[f] = take[k].mode;
            ((uint64_t*)(H + L.f_known))[f] = h->known.empty() ? 0 : h->known[k];
            if (nx) {                                                   // the checksum goes on, or ends in its digest
                (H + L.f_xmode)[f] = XXH_CARRY_IN | ((take[k].mode & WRITER_TAIL) ? 0 : XXH_CARRY_OUT);
                ((Xxh32Carry*)(H + L.f_xxh))[f] = h->st[k].xxh;
            }
            i += p_len[f] ? (p_len[f] + bs - 1) / bs : 1;
        }
        // p.f_len is the declared content size; the LZ4Block writer kernels do not read it
        const FramePlan P{ d_src, d_dst, s->d_slots,
                           (const uint64_t*)(D + L.b_soff), (const int32_t*)(D + L.b_slen), (const uint64_t*)(D + L.b_slot), (const int32_t*)(D + L.b_clen),
                           (uint64_t*)(D + L.b_poff), (int32_t*)(D + L.b_plen), (const uint32_t*)(D + L.b_sum),
                           (const uint32_t*)(D + L.i_frame), (const int32_t*)(D + L.i_block), (int32_t*)(D + L.i_size), (uint64_t*)(D + L.i_off),
                           (const uint64_t*)(D + L.f_known), (const uint32_t*)(D + L.f_sum), (uint64_t*)(D + L.f_off), (uint64_t*)(D + L.f_end),
                           (uint32_t)ni, frame ? h->code : 0, flags, frame ? 0 : h->code };
        const FrameWriterPlan W{ P, (const uint64_t*)(D + L.f_doff), (const uint32_t*)(D + L.f_first), (const uint8_t*)(D + L.f_mode) };

        Drain drain{ st, side->st };
        CK(cudaMemcpyAsync(D, H, L.bytes, cudaMemcpyHostToDevice, st));
        const bool early_sums = frame ? nx != 0 : nb > 0;
        if (early_sums) {           // checksums of the sources alone, so from the start, beside everything else
            CK(cudaEventRecord(side->fork, st));
            CK(cudaStreamWaitEvent(side->st, side->fork, 0));
            if (frame)
                CK(counted(launch_xxh32_long_carry(d_src, (const uint64_t*)(D + L.f_soff), (const uint64_t*)(D + L.f_len),
                                                   (uint32_t*)(D + L.f_sum), (Xxh32Carry*)(D + L.f_xxh), D + L.f_xmode, nf, side->st)));
            else
                CK(counted((taken / nb >= XXH_LONG_AVG ? launch_xxh32_long : launch_xxh32)(
                    d_src, P.b_soff, P.b_slen, LZ4BLOCK_SEED, (uint32_t*)P.b_sum, (size_t)nb, side->st)));
            CK(cudaEventRecord(side->join, side->st));
        }
        rc = chunk_loop(P, (const int32_t*)(D + L.b_ccap), s->d_slots, chunks, h->hc_level, (uint64_t*)(D + L.carry),
                        [&](uint32_t i0, uint32_t n) { return frame ? launch_frame_writer_sizes(W, i0, n, st)
                                                                     : launch_lz4block_writer_sizes(W, i0, n, st); },
                        [&](uint32_t i0, uint32_t n) { return frame ? launch_frame_writer_emit(W, i0, n, st)
                                                                     : launch_lz4block_writer_emit(W, i0, n, st); }, st);
        if (rc) return rc;
        if ((flags & 2) && nb) {    // block checksums over the payloads as written, as compress_blocks_dev takes them
            CK(counted((taken / nb >= XXH_LONG_AVG ? launch_xxh32_long : launch_xxh32)(
                d_dst, P.b_poff, P.b_plen, 0, (uint32_t*)P.b_sum, (size_t)nb, st)));
        }
        if (early_sums) CK(cudaStreamWaitEvent(st, side->join, 0));
        CK(counted(frame ? launch_frame_writer_seal(W, st) : launch_lz4block_writer_seal(W, st)));
        CK(cudaMemcpyAsync(H + L.f_off, D + L.f_off, L.bytes - L.f_off, cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        drain.done = true;
        for (size_t f = 0; f < nf; f++) range[p_stream[f]] = ((const uint64_t*)(H + L.f_end))[f] - ((const uint64_t*)(H + L.f_off))[f];
        if (nx) xxh.assign((const Xxh32Carry*)(H + L.f_xxh), (const Xxh32Carry*)(H + L.f_xxh) + nf);
    }
    for (size_t k = 0; k < ns; k++) {
        status[k] = take[k].status; src_consumed[k] = take[k].taken; produced[k] = range[k]; need[k] = take[k].need;
        if (take[k].mode & WRITER_HEAD) h->st[k].head = 1;
        if (take[k].status == B200LZ4F_DONE) h->st[k].done = 1;
    }
    for (size_t f = 0; f < xxh.size(); f++) h->st[p_stream[f]].xxh = xxh[f];
    return 0;
}

// A device writer, write(d_src, src_off, src_len, d_dst, capacity, st) for one source, run on a copy of src in the thread's
// staging buffer: the source at its own 16-byte phase (the fast compressor's chunks, and so its streams, follow the source's
// alignment), the container behind it.  bound: the container's size bound, checked against cap by the caller.
template <class Write>
static int64_t write_staged(const uint8_t* src, size_t n, uint8_t* dst, size_t bound, Write write)
{
    FrameScratch* s; cudaStream_t st;
    int rc = get_frame_scratch(&s, nullptr, &st); if (rc) return rc;
    const uint64_t phase = (uintptr_t)src & 15, len = n, at = (phase + n + 15) & ~uint64_t(15);
    rc = reserve_device(s->d_stage, s->stage_cap, at + bound); if (rc) return rc;
    Drain drain{ st };
    CK(cudaMemcpyAsync(s->d_stage + phase, src, n, cudaMemcpyHostToDevice, st));
    const int64_t w = write(s->d_stage, &phase, &len, s->d_stage + at, bound, st);
    if (w < 0) return w;
    CK(cudaMemcpyAsync(dst, s->d_stage + at, (size_t)w, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    drain.done = true;
    return w;
}

// ---------------------------------------------------------------- LZ4Block reader, streams in device memory (lz4block.cu)
// Where one call's per-stream arrays lie in the reader scratch's d_seg / h_seg: the inputs go up, the two block counts come
// back after the counting walk, the results (result, consumed, content) at the end.
struct Lz4BlockStreamLayout {
    size_t s_off, s_len, d_off, d_cap, n_comp, n_raw, tail, ip, p_comp, p_raw, totals, result, consumed, content, bytes = 0;
    explicit Lz4BlockStreamLayout(size_t ns)
    {
        auto take = [&](size_t n) { const size_t at = bytes; bytes = (bytes + n + 15) & ~size_t(15); return at; };
        s_off = take(8 * ns); s_len = take(8 * ns); d_off = take(8 * ns); d_cap = take(8 * ns);
        n_comp = take(4 * ns); n_raw = take(4 * ns); tail = take(4 * ns); ip = take(8 * ns); p_comp = take(8 * ns); p_raw = take(8 * ns);
        totals = take(16);
        result = take(8 * ns); consumed = take(8 * ns); content = take(8 * ns);
    }
};
// ... and the records of nc compressed and nr stored blocks in d_recs; they never leave the device
struct Lz4BlockRecLayout {
    size_t c_soff, c_doff, c_clen, c_olen, c_res, r_soff, r_doff, r_len, b_doff, b_len, b_comp, b_want, b_sum, bytes = 0;
    Lz4BlockRecLayout(size_t nc, size_t nr)
    {
        auto take = [&](size_t n) { const size_t at = bytes; bytes = (bytes + n + 15) & ~size_t(15); return at; };
        const size_t nb = nc + nr;
        c_soff = take(8 * nc); c_doff = take(8 * nc); c_clen = take(4 * nc); c_olen = take(4 * nc); c_res = take(4 * nc);
        r_soff = take(8 * nr); r_doff = take(8 * nr); r_len = take(4 * nr);
        b_doff = take(8 * nb); b_len = take(4 * nb); b_comp = take(4 * nb); b_want = take(4 * nb); b_sum = take(4 * nb);
    }
};

// Points r's record arrays into the call's record region B.
static void bind_lz4block_records(Lz4BlockRead& r, uint8_t* B, const Lz4BlockRecLayout& R)
{
    r.c_soff = (uint64_t*)(B + R.c_soff); r.c_doff = (uint64_t*)(B + R.c_doff);
    r.c_clen = (int32_t*)(B + R.c_clen); r.c_olen = (int32_t*)(B + R.c_olen); r.c_res = (int32_t*)(B + R.c_res);
    r.r_soff = (uint64_t*)(B + R.r_soff); r.r_doff = (uint64_t*)(B + R.r_doff); r.r_len = (int32_t*)(B + R.r_len);
    r.b_doff = (uint64_t*)(B + R.b_doff); r.b_len = (int32_t*)(B + R.b_len); r.b_comp = (int32_t*)(B + R.b_comp);
    r.b_want = (uint32_t*)(B + R.b_want); r.b_sum = (uint32_t*)(B + R.b_sum);
}

// The payload launches behind a recording walk: the stored blocks gathered and the compressed ones decoded straight into
// d_dst, then the XXH32 of every decoded block.  bytes / room: the call's source bytes and room; nc / nr: its compressed /
// stored blocks.
static int lz4block_payload_launches(const Lz4BlockRead& r, uint8_t* d_dst, uint64_t bytes, uint64_t room, uint64_t nc,
                                     uint64_t nr, cudaStream_t st)
{
    const uint64_t nb = nc + nr;
    if (nr) CK(counted(launch_gather(r.src, r.r_soff, r.r_len, d_dst, r.r_doff, (size_t)nr, st)));
    if (nc) {                       // as the host reader: src_avail = the compressed length, dst_len = the original length
        const BatchArgs a{ r.src, r.c_soff, r.c_clen, d_dst, r.c_doff, r.c_olen, r.c_res, (size_t)nc };
        CK(counted(launch_decompress_fast(a, st)));
    }
    if (nb) {                       // the decoded bytes are at most the room given, and at most 255 per source byte
        const uint64_t decoded = room < bytes * 255 ? room : bytes * 255;
        CK(counted((decoded / nb >= XXH_LONG_AVG ? launch_xxh32_long : launch_xxh32)(d_dst, r.b_doff, r.b_len, LZ4BLOCK_SEED,
                                                                                      r.b_sum, (size_t)nb, st)));
    }
    return 0;
}

// Counting walk, two scans of the counts (only their totals come to the host: the records' room), recording walk, then
// the blocks decode straight into d_dst, their checksums, and one verdict per stream.  The launches do not depend on the
// number of streams or blocks.
static int lz4block_decompress_dev(const uint8_t* d_src, const uint64_t* src_off, const uint64_t* src_len, size_t ns,
                                   uint8_t* d_dst, const uint64_t* dst_off, const uint64_t* dst_cap, bool stop,
                                   int64_t* result, uint64_t* src_consumed, uint64_t* content_len, cudaStream_t st)
{
    if (ns == 0) return 0;
    if (!src_off || !src_len || !dst_off || !dst_cap || !result) return fail_arg("null pointer");
    if (ns > 0x7FFFFFFFull) return fail_arg("too many streams in one call");
    uint64_t bytes, room;
    int rc = check_stream_ranges(ns, src_len, 1ull << 47, dst_off, dst_cap, d_src, d_dst, bytes, room);
    if (rc) return rc;
    if (bytes / LZ4BLOCK_HEADER > 0x7FFFFFFFull) return fail_arg("too many blocks in one call");
    FrameReadScratch* s;
    rc = get_frame_read_scratch(&s);
    const Lz4BlockStreamLayout L(ns);
    if (!rc) rc = reserve_device(s->d_seg, s->seg_cap, L.bytes);
    if (!rc) rc = reserve_pinned(s->h_seg, s->h_seg_cap, L.bytes);
    if (rc) return rc;
    uint8_t *D = s->d_seg, *H = s->h_seg;
    memcpy(H + L.s_off, src_off, 8 * ns); memcpy(H + L.s_len, src_len, 8 * ns);
    memcpy(H + L.d_off, dst_off, 8 * ns); memcpy(H + L.d_cap, dst_cap, 8 * ns);
    Lz4BlockRead r{};
    r.src = d_src;
    r.s_off = (const uint64_t*)(D + L.s_off); r.s_len = (const uint64_t*)(D + L.s_len);
    r.d_off = (const uint64_t*)(D + L.d_off); r.d_cap = (const uint64_t*)(D + L.d_cap);
    r.n_comp = (int32_t*)(D + L.n_comp); r.n_raw = (int32_t*)(D + L.n_raw); r.tail = (int32_t*)(D + L.tail);
    r.ip = (uint64_t*)(D + L.ip); r.content = (uint64_t*)(D + L.content);
    r.p_comp = (const uint64_t*)(D + L.p_comp); r.p_raw = (const uint64_t*)(D + L.p_raw);
    r.result = (int64_t*)(D + L.result); r.consumed = (uint64_t*)(D + L.consumed);
    r.ns = (uint32_t)ns; r.stop = stop;
    uint64_t* totals = (uint64_t*)(D + L.totals);

    Drain drain{ st };
    CK(cudaMemcpyAsync(D, H, L.n_comp, cudaMemcpyHostToDevice, st));
    g_launch_count.fetch_add(3, std::memory_order_relaxed);
    CK(launch_lz4block_walk(r, false, st));
    CK(launch_scan(r.n_comp, (uint64_t*)r.p_comp, totals, nullptr, ns, st));
    CK(launch_scan(r.n_raw, (uint64_t*)r.p_raw, totals + 1, nullptr, ns, st));
    CK(cudaMemcpyAsync(H + L.totals, totals, 16, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    const uint64_t nc = ((const uint64_t*)(H + L.totals))[0], nr = ((const uint64_t*)(H + L.totals))[1];
    const Lz4BlockRecLayout R(nc, nr);
    rc = reserve_device(s->d_recs, s->recs_cap, R.bytes + 16); if (rc) return rc;
    bind_lz4block_records(r, s->d_recs, R);
    CK(counted(launch_lz4block_walk(r, true, st)));
    rc = lz4block_payload_launches(r, d_dst, bytes, room, nc, nr, st); if (rc) return rc;
    CK(counted(launch_lz4block_verdict(r, st)));
    CK(cudaMemcpyAsync(H + L.result, D + L.result, L.bytes - L.result, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    drain.done = true;
    memcpy(result, H + L.result, 8 * ns);
    if (src_consumed) memcpy(src_consumed, H + L.consumed, 8 * ns);
    if (content_len) memcpy(content_len, H + L.content, 8 * ns);
    return 0;
}

// ---- the incremental LZ4Block reader (b200lz4block_reader_*; kernels: lz4block.cu).  The reader is host data: per stream
// its latched status (0 while reading, B200LZ4F_DONE, or -1 / -2).
struct Lz4BlockReaderHandle {
    size_t ns; bool stop;
    std::vector<int32_t> st;
};
// One call's per-stream arrays in the reader scratch's d_seg / h_seg: the arguments and states go up, the scan totals come
// back after the counting walk, the results at the end.
struct Lz4BlockReaderLayout {
    size_t s_off, s_len, d_off, d_cap, eof, st_in, totals, n_comp, n_raw, tail, p_comp, p_raw, status, consumed, produced, need,
           bytes = 0;
    explicit Lz4BlockReaderLayout(size_t ns)
    {
        auto take = [&](size_t n) { const size_t at = bytes; bytes = (bytes + n + 15) & ~size_t(15); return at; };
        s_off = take(8 * ns); s_len = take(8 * ns); d_off = take(8 * ns); d_cap = take(8 * ns); eof = take(ns); st_in = take(4 * ns);
        totals = take(16);
        n_comp = take(4 * ns); n_raw = take(4 * ns); tail = take(4 * ns); p_comp = take(8 * ns); p_raw = take(8 * ns);
        status = take(4 * ns); consumed = take(8 * ns); produced = take(8 * ns); need = take(8 * ns);
    }
};

// lz4block_decompress_dev's steps from each stream's latched status, with the walk resumable and the room applied by it:
// counting walk, two scans (their totals come to the host, to size the records), recording walk, the blocks decode straight
// into d_dst, their checksums, one verdict warp per stream.  The launches do not depend on the number of streams or blocks.
static int lz4block_reader_read_dev(Lz4BlockReaderHandle* h, const uint8_t* d_src, const uint64_t* src_off, const uint64_t* src_len,
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
    if (bytes / LZ4BLOCK_HEADER > 0x7FFFFFFFull) return fail_arg("too many blocks in one call");
    FrameReadScratch* s;
    rc = get_frame_read_scratch(&s);
    const Lz4BlockReaderLayout L(ns);
    if (!rc) rc = reserve_device(s->d_seg, s->seg_cap, L.bytes);
    if (!rc) rc = reserve_pinned(s->h_seg, s->h_seg_cap, L.bytes);
    if (rc) return rc;
    uint8_t *D = s->d_seg, *H = s->h_seg;
    memcpy(H + L.s_off, src_off, 8 * ns); memcpy(H + L.s_len, src_len, 8 * ns);
    memcpy(H + L.d_off, dst_off, 8 * ns); memcpy(H + L.d_cap, dst_cap, 8 * ns); memcpy(H + L.eof, eof, ns);
    memcpy(H + L.st_in, h->st.data(), 4 * ns);
    Lz4BlockReaderRead q{};
    Lz4BlockRead& r = q.r;
    r.src = d_src;
    r.s_off = (const uint64_t*)(D + L.s_off); r.s_len = (const uint64_t*)(D + L.s_len);
    r.d_off = (const uint64_t*)(D + L.d_off); r.d_cap = (const uint64_t*)(D + L.d_cap);
    r.n_comp = (int32_t*)(D + L.n_comp); r.n_raw = (int32_t*)(D + L.n_raw); r.tail = (int32_t*)(D + L.tail);
    r.p_comp = (const uint64_t*)(D + L.p_comp); r.p_raw = (const uint64_t*)(D + L.p_raw);
    r.consumed = (uint64_t*)(D + L.consumed);
    r.ns = (uint32_t)ns; r.stop = h->stop;
    q.eof = D + L.eof; q.st_in = (const int32_t*)(D + L.st_in);
    q.status = (int32_t*)(D + L.status); q.produced = (uint64_t*)(D + L.produced); q.need = (uint64_t*)(D + L.need);
    uint64_t* totals = (uint64_t*)(D + L.totals);

    Drain drain{ st };
    CK(cudaMemcpyAsync(D, H, L.totals, cudaMemcpyHostToDevice, st));
    g_launch_count.fetch_add(3, std::memory_order_relaxed);
    CK(launch_lz4block_reader_walk(q, false, st));
    CK(launch_scan(r.n_comp, (uint64_t*)r.p_comp, totals, nullptr, ns, st));
    CK(launch_scan(r.n_raw, (uint64_t*)r.p_raw, totals + 1, nullptr, ns, st));
    CK(cudaMemcpyAsync(H + L.totals, totals, 16, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    const uint64_t nc = ((const uint64_t*)(H + L.totals))[0], nr = ((const uint64_t*)(H + L.totals))[1], nb = nc + nr;
    // the whole-stream reader's records, then per block where its unit starts
    const Lz4BlockRecLayout R(nc, nr);
    const size_t k_at = (R.bytes + 15) & ~size_t(15);
    rc = reserve_device(s->d_recs, s->recs_cap, k_at + 8 * nb + 16); if (rc) return rc;
    bind_lz4block_records(r, s->d_recs, R);
    q.k_at = (uint64_t*)(s->d_recs + k_at);
    CK(counted(launch_lz4block_reader_walk(q, true, st)));
    rc = lz4block_payload_launches(r, d_dst, bytes, room, nc, nr, st); if (rc) return rc;
    CK(counted(launch_lz4block_reader_verdict(q, st)));
    CK(cudaMemcpyAsync(H + L.status, D + L.status, L.bytes - L.status, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    drain.done = true;
    memcpy(status, H + L.status, 4 * ns);
    memcpy(src_consumed, H + L.consumed, 8 * ns);
    memcpy(produced, H + L.produced, 8 * ns);
    memcpy(need, H + L.need, 8 * ns);
    for (size_t k = 0; k < ns; k++)
        if (status[k] < 0 || status[k] == B200LZ4F_DONE) h->st[k] = status[k];
    return 0;
}

// ---------------------------------------------------------------- length-prefixed records in device memory (with_length.cu)
// Where one call's per-record arrays lie in the reader scratch's d_seg / h_seg: the arguments go up, the results come back,
// the decoder's arguments and results stay on the device.
struct WithLengthLayout {
    size_t s_off, s_len, d_off, d_cap, b_soff, b_slen, b_dlen, b_res, head, result, orig, bytes = 0;
    explicit WithLengthLayout(size_t n)
    {
        auto take = [&](size_t k) { const size_t at = bytes; bytes = (bytes + k + 15) & ~size_t(15); return at; };
        s_off = take(8 * n); s_len = take(8 * n); d_off = take(8 * n); d_cap = take(8 * n);
        b_soff = take(8 * n); b_slen = take(4 * n); b_dlen = take(4 * n); b_res = take(4 * n); head = take(4 * n);
        result = take(8 * n); orig = take(8 * n);
    }
};

// The header kernel, the fast or safe decoder over every record, the verdict kernel: three launches whatever n is, and one
// synchronisation.
static int with_length_decompress_dev(const uint8_t* d_src, const uint64_t* src_off, const uint64_t* src_len, size_t n,
                                      uint8_t* d_dst, const uint64_t* dst_off, const uint64_t* dst_cap, bool safe,
                                      int64_t* result, int64_t* orig_len, cudaStream_t st)
{
    if (n == 0) return 0;
    if (!src_off || !src_len || !dst_off || !dst_cap || !result) return fail_arg("null pointer");
    if (n > 0x7FFFFFFFull) return fail_arg("too many records in one call");
    uint64_t bytes, room;                                           // a record is at most 2^31 - 1 bytes
    int rc = check_stream_ranges(n, src_len, 0x7FFFFFFFull, dst_off, dst_cap, d_src, d_dst, bytes, room);
    if (rc) return rc;
    FrameReadScratch* s;
    rc = get_frame_read_scratch(&s);
    const WithLengthLayout L(n);
    if (!rc) rc = reserve_device(s->d_seg, s->seg_cap, L.bytes);
    if (!rc) rc = reserve_pinned(s->h_seg, s->h_seg_cap, L.bytes);
    if (rc) return rc;
    uint8_t *D = s->d_seg, *H = s->h_seg;
    memcpy(H + L.s_off, src_off, 8 * n); memcpy(H + L.s_len, src_len, 8 * n);
    memcpy(H + L.d_off, dst_off, 8 * n); memcpy(H + L.d_cap, dst_cap, 8 * n);
    WithLengthRead r{};
    r.src = d_src;
    r.s_off = (const uint64_t*)(D + L.s_off); r.s_len = (const uint64_t*)(D + L.s_len); r.d_cap = (const uint64_t*)(D + L.d_cap);
    r.b_soff = (uint64_t*)(D + L.b_soff); r.b_slen = (int32_t*)(D + L.b_slen); r.b_dlen = (int32_t*)(D + L.b_dlen);
    r.b_res = (int32_t*)(D + L.b_res); r.head = (int32_t*)(D + L.head);
    r.result = (int64_t*)(D + L.result); r.orig_len = (int64_t*)(D + L.orig);
    r.n = (uint32_t)n; r.safe = safe;
    // fast: src_len = the readable bytes, dst_cap = the exact decoded size; safe: the block's size and maxDestLen
    const BatchArgs a{ d_src, r.b_soff, r.b_slen, d_dst, (const uint64_t*)(D + L.d_off), r.b_dlen, r.b_res, n };

    Drain drain{ st };
    CK(cudaMemcpyAsync(D, H, L.b_soff, cudaMemcpyHostToDevice, st));
    g_launch_count.fetch_add(3, std::memory_order_relaxed);
    CK(launch_with_length_head(r, st));
    CK(safe ? launch_decompress_safe(a, st) : launch_decompress_fast(a, st));
    CK(launch_with_length_verdict(r, st));
    CK(cudaMemcpyAsync(H + L.result, D + L.result, L.bytes - L.result, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    drain.done = true;
    memcpy(result, H + L.result, 8 * n);
    if (orig_len) memcpy(orig_len, H + L.orig, 8 * n);
    return 0;
}

// The host reader's sink of walk_lz4block: the stored blocks that fit are copied at once, the compressed ones and every
// checksum go to the batch calls afterwards.
struct Lz4BlockHostSink {
    const uint8_t* src; uint8_t* dst; Lz4BlockRoom room;
    std::vector<uint64_t> soff, doff, hoff; std::vector<int32_t> savail, dlen, hlen; std::vector<uint32_t> want;
    void block(uint64_t at, bool raw, int32_t clen, int32_t olen, uint32_t check)
    {
        const uint64_t op = room.used;
        if (!room.take(olen)) return;
        if (raw) memcpy(dst + op, src + at, (size_t)olen);
        else { soff.push_back(at); savail.push_back(clen); doff.push_back(op); dlen.push_back(olen); }
        hoff.push_back(op); hlen.push_back(olen); want.push_back(check);
    }
};

} // namespace b200

extern "C" {

size_t b200lz4f_compress_bound(size_t n, int bsCode)
{
    if (bsCode < 4 || bsCode > 7) return 0;
    const size_t bs = (size_t)1 << (8 + 2 * bsCode), nb = (n + bs - 1) / bs;
    return 4 + 2 + 8 + 1 + nb * 8 + n + 4 + 4;
}

int64_t b200lz4f_compress_dev(const uint8_t* d_src, const uint64_t* src_off, const uint64_t* src_len, size_t nf,
                              uint8_t* d_dst, size_t dst_capacity, uint64_t* frame_off, uint64_t* frame_len,
                              int bsCode, int flags, int hc_level, void* stream)
{
    return b200::compress_frames_dev(d_src, src_off, src_len, nf, d_dst, dst_capacity, frame_off, frame_len, bsCode, flags,
                                     hc_level, (cudaStream_t)stream);
}

// The device writer on a staged copy of src (write_staged)
int64_t b200lz4f_compress_host_hc(const uint8_t* src, size_t n, uint8_t* dst, size_t cap, int bsCode, int flags, int hc_level)
{
    if (bsCode < 4 || bsCode > 7) return b200::fail_arg("bsCode must be 4..7");
    const size_t bound = b200lz4f_compress_bound(n, bsCode);
    if (cap < bound) return -9;
    return b200::write_staged(src, n, dst, bound, [&](const uint8_t* d_src, const uint64_t* off, const uint64_t* len, uint8_t* d_dst,
                                                      size_t room, cudaStream_t st) {
        return b200::compress_frames_dev(d_src, off, len, 1, d_dst, room, nullptr, nullptr, bsCode, flags, hc_level, st);
    });
}
int64_t b200lz4f_compress_host(const uint8_t* src, size_t n, uint8_t* dst, size_t cap, int bsCode, int flags)
{ return b200lz4f_compress_host_hc(src, n, dst, cap, bsCode, flags, 0); }

// the incremental writer (writer_write_dev): host data only, no CUDA call in create or free
void* b200lz4f_writer_create(size_t ns, int bsCode, int flags, int hc_level, const int64_t* known_size, int* err)
{
    if (err) *err = 0;
    auto fail = [&](const char* what) -> void* { const int rc = b200::fail_arg(what); if (err) *err = rc; return nullptr; };
    if (bsCode < 4 || bsCode > 7) return fail("bsCode must be 4..7");
    if (ns > 0x7FFFFFFFull) return fail("too many streams in one writer");
    if (flags & 4) {                // LZ4FrameOutputStream's constructor: a declared size needs a known one (:138-140)
        if (ns && !known_size) return fail("known_size is needed with flags bit 2");
        for (size_t k = 0; k < ns; k++) if (known_size[k] < 0) return fail("known_size must be >= 0");
    }
    void* h = b200::new_writer(b200::Container::Frame, ns, 1ull << (8 + 2 * bsCode), bsCode, flags, hc_level,
                               (flags & 4) ? known_size : nullptr);
    return h ? h : fail("out of host memory");
}

int b200lz4f_writer_write_dev(void* writer, const uint8_t* d_src, const uint64_t* src_off, const uint64_t* src_len,
                              const uint8_t* op, uint8_t* d_dst, const uint64_t* dst_off, const uint64_t* dst_cap,
                              int32_t* status, uint64_t* src_consumed, uint64_t* produced, uint64_t* need, void* stream)
{
    return b200::writer_write_dev((b200::WriterHandle*)writer, d_src, src_off, src_len, op, d_dst, dst_off, dst_cap, status,
                                  src_consumed, produced, need, (cudaStream_t)stream);
}

void b200lz4f_writer_free(void* writer) { delete (b200::WriterHandle*)writer; }

// ---------------------------------------------------------------- "LZ4Block" container
size_t b200lz4block_compress_bound(size_t n, int blockSize)
{
    if (blockSize < 64 || blockSize > (1 << 25)) return 0;
    const size_t nb = (n + blockSize - 1) / blockSize;
    return (nb + 1) * b200::LZ4BLOCK_HEADER + n + nb * 16 + n / 255;
}

int64_t b200lz4block_compress_dev(const uint8_t* d_src, const uint64_t* src_off, const uint64_t* src_len, size_t ns,
                                  uint8_t* d_dst, size_t dst_capacity, uint64_t* stream_off, uint64_t* stream_len,
                                  int blockSize, int hc_level, void* stream)
{
    return b200::compress_lz4block_dev(d_src, src_off, src_len, ns, d_dst, dst_capacity, stream_off, stream_len, blockSize,
                                       hc_level, (cudaStream_t)stream);
}

// The device writer on a staged copy of src (write_staged)
int64_t b200lz4block_compress_host_hc(const uint8_t* src, size_t n, uint8_t* dst, size_t cap, int blockSize, int hc_level)
{
    if (blockSize < 64 || blockSize > (1 << 25)) return b200::fail_arg("blockSize must be 64..32 MiB");
    const size_t bound = b200lz4block_compress_bound(n, blockSize);
    if (cap < bound) return -9;
    return b200::write_staged(src, n, dst, bound, [&](const uint8_t* d_src, const uint64_t* off, const uint64_t* len, uint8_t* d_dst,
                                                      size_t room, cudaStream_t st) {
        return b200::compress_lz4block_dev(d_src, off, len, 1, d_dst, room, nullptr, nullptr, blockSize, hc_level, st);
    });
}
int64_t b200lz4block_compress_host(const uint8_t* src, size_t n, uint8_t* dst, size_t cap, int blockSize)
{ return b200lz4block_compress_host_hc(src, n, dst, cap, blockSize, 0); }

// Decodes an LZ4Block stream the way LZ4BlockInputStream reads it.  stopOnEmptyBlock != 0 (the reference's default, :100-104):
// reading ends at the first empty block, whatever follows is left alone (*srcConsumed says where), and a stream that ends
// before one is "Stream ended prematurely" (:192-198).  stopOnEmptyBlock == 0: empty blocks are stepped over, concatenated
// streams continue, and the end of src at (or inside) a header ends the stream quietly (:193-194, tryReadFully).
// Returns decoded bytes; -1 premature end, -2 "Stream is corrupted", -9 dst too small.
int64_t b200lz4block_decompress_host(const uint8_t* src, size_t n, uint8_t* dst, size_t cap, int stopOnEmptyBlock, size_t* srcConsumed)
{
    b200::Lz4BlockHostSink sink{ src, dst, b200::Lz4BlockRoom{ cap } };
    const b200::Lz4BlockEnd e = b200::walk_lz4block(src, n, stopOnEmptyBlock != 0, sink);   // refill (:191-264)
    // what is wrong with the container itself, behind the blocks taken: the reader would have decoded and checked THOSE
    // first, so their verdict comes first.  A block that does not fit lies before anything the walk met later.
    const int64_t tail = sink.room.full ? -9 : e.err;
    // per block the reader decodes, compares the consumed length, then the checksum -- all "Stream is corrupted" (:236-262)
    if (!sink.soff.empty()) {
        std::vector<int32_t> res(sink.soff.size());
        int rc = b200lz4_decompress_fast_batch_host(src, sink.soff.data(), sink.savail.data(), dst, sink.doff.data(), sink.dlen.data(),
                                                    res.data(), sink.soff.size());
        if (rc) return rc;
        for (size_t i = 0; i < res.size(); i++) if (res[i] != sink.savail[i]) return -2;   // compressedLen != compressedLen2 (:247-250)
    }
    if (!sink.hoff.empty()) {
        std::vector<uint32_t> sums(sink.hoff.size());
        int rc = b200xxh32_batch_host(dst, sink.hoff.data(), sink.hlen.data(), b200::LZ4BLOCK_SEED, sums.data(), sink.hoff.size());
        if (rc) return rc;
        for (size_t i = 0; i < sums.size(); i++) if ((sums[i] & 0x0FFFFFFFu) != sink.want[i]) return -2;
    }
    if (tail) return tail;
    if (srcConsumed) *srcConsumed = e.ip;
    return (int64_t)sink.room.used;
}

int b200lz4block_decompress_dev(const uint8_t* d_src, const uint64_t* src_off, const uint64_t* src_len, size_t ns,
                                uint8_t* d_dst, const uint64_t* dst_off, const uint64_t* dst_cap, int stopOnEmptyBlock,
                                int64_t* result, uint64_t* src_consumed, uint64_t* content_len, void* stream)
{
    return b200::lz4block_decompress_dev(d_src, src_off, src_len, ns, d_dst, dst_off, dst_cap, stopOnEmptyBlock != 0, result,
                                         src_consumed, content_len, (cudaStream_t)stream);
}

// the incremental writer and reader (writer_write_dev, lz4block_reader_read_dev): host data only, no CUDA call in
// create or free
void* b200lz4block_writer_create(size_t ns, int blockSize, int hc_level, int* err)
{
    if (err) *err = 0;
    auto fail = [&](const char* what) -> void* { const int rc = b200::fail_arg(what); if (err) *err = rc; return nullptr; };
    if (blockSize < 64 || blockSize > (1 << 25)) return fail("blockSize must be 64..32 MiB");
    if (ns > 0x7FFFFFFFull) return fail("too many streams in one writer");
    void* h = b200::new_writer(b200::Container::LZ4Block, ns, (uint64_t)blockSize, b200::lz4block_level(blockSize), 0, hc_level,
                               nullptr);
    return h ? h : fail("out of host memory");
}

int b200lz4block_writer_write_dev(void* writer, const uint8_t* d_src, const uint64_t* src_off, const uint64_t* src_len,
                                  const uint8_t* op, uint8_t* d_dst, const uint64_t* dst_off, const uint64_t* dst_cap,
                                  int32_t* status, uint64_t* src_consumed, uint64_t* produced, uint64_t* need, void* stream)
{
    return b200::writer_write_dev((b200::WriterHandle*)writer, d_src, src_off, src_len, op, d_dst, dst_off, dst_cap, status,
                                  src_consumed, produced, need, (cudaStream_t)stream);
}

void b200lz4block_writer_free(void* writer) { delete (b200::WriterHandle*)writer; }

void* b200lz4block_reader_create(size_t ns, int stopOnEmptyBlock, int* err)
{
    if (err) *err = 0;
    auto fail = [&](const char* what) -> void* { const int rc = b200::fail_arg(what); if (err) *err = rc; return nullptr; };
    if (ns > 0x7FFFFFFFull) return fail("too many streams in one reader");
    b200::Lz4BlockReaderHandle* h = new (std::nothrow) b200::Lz4BlockReaderHandle;
    if (!h) return fail("out of host memory");
    h->ns = ns; h->stop = stopOnEmptyBlock != 0;
    try { h->st.assign(ns, 0); }
    catch (...) { delete h; return fail("out of host memory"); }
    return h;
}

int b200lz4block_reader_read_dev(void* reader, const uint8_t* d_src, const uint64_t* src_off, const uint64_t* src_len,
                                 const uint8_t* eof, uint8_t* d_dst, const uint64_t* dst_off, const uint64_t* dst_cap,
                                 int32_t* status, uint64_t* src_consumed, uint64_t* produced, uint64_t* need, void* stream)
{
    return b200::lz4block_reader_read_dev((b200::Lz4BlockReaderHandle*)reader, d_src, src_off, src_len, eof, d_dst, dst_off,
                                          dst_cap, status, src_consumed, produced, need, (cudaStream_t)stream);
}

void b200lz4block_reader_free(void* reader) { delete (b200::Lz4BlockReaderHandle*)reader; }

// ---------------------------------------------------------------- length-prefixed block (LZ4CompressorWithLength.java:45-50)
int b200lz4_compress_with_length(const char* src, char* dst, int srcSize, int dstCapacity)
{
    if (dstCapacity < 4) return 0;
    const int r = b200lz4_compress_default(src, dst + 4, srcSize, dstCapacity - 4);
    if (r <= 0) return r;
    put32((uint8_t*)dst, (uint32_t)srcSize);
    return r + 4;
}
int b200lz4_decompressed_length(const char* src) { return (int)get32((const uint8_t*)src); }   // LZ4DecompressorWithLength.java:52-54
// fast-decompressor flavour: returns bytes read (incl. the 4-byte prefix) or < 0 (LZ4DecompressorWithLength.java:125-131)
int b200lz4_decompress_with_length(const char* src, int srcAvail, char* dst, int dstCapacity)
{
    if (srcAvail < 4) return -1;
    const int n = b200lz4_decompressed_length(src);
    if (n < 0 || n > dstCapacity) return -1;
    const int r = b200lz4_decompress_fast_bounded(src + 4, srcAvail - 4, dst, n);
    return r < 0 ? r : r + 4;
}
// safe-decompressor flavour (lz4-java 1.8): src is exactly one record; returns the bytes decoded or < 0
// (LZ4DecompressorWithLength.java:148-154)
int b200lz4_decompress_with_length_safe(const char* src, int srcLen, char* dst, int dstCapacity)
{
    if (srcLen < 4) return -1;
    const int n = b200lz4_decompressed_length(src);
    if (n < 0 || n > dstCapacity) return -1;
    return b200lz4_decompress_safe(src + 4, dst, srcLen - 4, n);
}

int64_t b200lz4_compress_with_length_dev(const uint8_t* d_src, const uint64_t* src_off, const uint64_t* src_len, size_t n,
                                         uint8_t* d_dst, size_t dst_capacity, uint64_t* rec_off, uint64_t* rec_len,
                                         int hc_level, void* stream)
{
    return b200::compress_with_length_dev(d_src, src_off, src_len, n, d_dst, dst_capacity, rec_off, rec_len, hc_level,
                                          (cudaStream_t)stream);
}

int b200lz4_decompress_with_length_dev(const uint8_t* d_src, const uint64_t* src_off, const uint64_t* src_len, size_t n,
                                       uint8_t* d_dst, const uint64_t* dst_off, const uint64_t* dst_cap, int safe,
                                       int64_t* result, int64_t* orig_len, void* stream)
{
    return b200::with_length_decompress_dev(d_src, src_off, src_len, n, d_dst, dst_off, dst_cap, safe != 0, result, orig_len,
                                            (cudaStream_t)stream);
}

} // extern "C"
