// kernels.h — internal launch interface between the C-ABI layer (capi.cu) and the kernels.
#pragma once
#include <atomic>
#include <cstddef>
#include <cstdint>
#ifdef B200_HOST_SIM
#include "simt.h"
#else
#include <cuda_runtime.h>
#endif

namespace b200 {

// One batch of independent LZ4 blocks (or hash buffers); every pointer is a device pointer.
struct BatchArgs {
    const uint8_t*  src_base;
    const uint64_t* src_off;
    const int32_t*  src_len;    // compress: bytes to compress; safe: compressed size; fast: readable bytes
    uint8_t*        dst_base;
    const uint64_t* dst_off;
    const int32_t*  dst_cap;    // compress/safe: capacity; fast: exact decoded size
    int32_t*        result;
    size_t          n;
};

cudaError_t launch_decompress_safe(const BatchArgs& a, cudaStream_t st);
cudaError_t launch_decompress_fast(const BatchArgs& a, cudaStream_t st);
cudaError_t launch_compress_fast(const BatchArgs& a, int max_src_len, cudaStream_t st);
cudaError_t launch_compress_hc(const BatchArgs& a, int level, cudaStream_t st);
cudaError_t launch_xxh32(const uint8_t* base, const uint64_t* off, const int32_t* len, uint32_t seed,
                         uint32_t* out, size_t n, cudaStream_t st);
// One warp per buffer: for a few long streams (frame content checksums).
cudaError_t launch_xxh32_long(const uint8_t* base, const uint64_t* off, const int32_t* len, uint32_t seed,
                              uint32_t* out, size_t n, cudaStream_t st);
// frame content checksums chained to the block decoder (frame.cu): one warp per frame follows the decoder's result words
static constexpr int32_t FRAME_RES_PENDING = int32_t(0x80808080);      // what cudaMemset(0x80) leaves; no decoder result looks like it
// A content checksum carried from call to call (the incremental reader, frame_reader.cu): XXH32's four lanes, the bytes of
// an unfinished stripe and the length so far.
struct Xxh32Carry { uint64_t total; uint32_t v[4]; uint8_t mem[16]; uint32_t memsize, pad; };
enum { XXH_CARRY_IN = 1, XXH_CARRY_OUT = 2 };   // mode[f]: start from carry[f]; leave the state in carry[f] instead of out[f]
// every frame starts fresh and ends in its digest
cudaError_t launch_xxh32_frames_chained(const uint8_t* slots, const uint64_t* blk_off, const uint32_t* f_first, const uint32_t* f_nblk,
                                        const int32_t* blk_comp, const int32_t* blk_rawlen, const int32_t* c_res,
                                        uint32_t* out, size_t n, cudaStream_t st);
// the same with a carried state per frame (mode: XXH_CARRY_* per frame); one launcher for both builds (B200_LAUNCH)
cudaError_t launch_xxh32_frames_chained_carry(const uint8_t* slots, const uint64_t* blk_off, const uint32_t* f_first,
                                              const uint32_t* f_nblk, const int32_t* blk_comp, const int32_t* blk_rawlen,
                                              const int32_t* c_res, uint32_t* out, size_t n, Xxh32Carry* carry,
                                              const uint8_t* mode, cudaStream_t st);
cudaError_t launch_xxh64(const uint8_t* base, const uint64_t* off, const int32_t* len, uint64_t seed,
                         uint64_t* out, size_t n, cudaStream_t st);
// launch_xxh32_long (seed 0) with 64-bit lengths and a carried state per run (the incremental writer, frame_writer.cu): run r
// is len[r] bytes at base + off[r]; mode[r] XXH_CARRY_IN starts from carry[r] (else a fresh state), XXH_CARRY_OUT leaves the
// state in carry[r] (else the digest goes to out[r]).  One warp per run; one launcher for both builds (B200_LAUNCH).
cudaError_t launch_xxh32_long_carry(const uint8_t* base, const uint64_t* off, const uint64_t* len, uint32_t* out, Xxh32Carry* carry,
                                    const uint8_t* mode, size_t n, cudaStream_t st);

// streaming hash: one device-resident state per handle, updated by a single-warp kernel
struct Xxh32State { uint64_t total; uint32_t v[4]; uint8_t mem[16]; uint32_t memsize; uint32_t seed; uint32_t digest; };
struct Xxh64State { uint64_t total; uint64_t v[4]; uint8_t mem[32]; uint32_t memsize; uint32_t pad; uint64_t seed; uint64_t digest; };
cudaError_t launch_xxh32_stream(Xxh32State* st, int op, uint32_t seed, const uint8_t* data, size_t len, cudaStream_t s);
cudaError_t launch_xxh64_stream(Xxh64State* st, int op, uint64_t seed, const uint8_t* data, size_t len, cudaStream_t s);
enum { XXH_OP_RESET = 0, XXH_OP_UPDATE = 1, XXH_OP_DIGEST = 2 };

cudaError_t launch_xxh64_long(const uint8_t* base, const uint64_t* off, const int32_t* len, uint64_t seed,
                              uint64_t* out, size_t n, cudaStream_t st);

// prefix-sum compaction of variable-length outputs (compact_host path)
cudaError_t launch_compact(const uint8_t* slots, const uint64_t* slot_off, const int32_t* lens,
                           uint8_t* out, uint64_t* out_off, uint64_t* total, size_t n, cudaStream_t st);
// the scan alone: out_off[i] = *carry_in + exclusive prefix of max(lens, 0); *total = *carry_in + the sum (carry_in may be
// NULL: 0).  carry_in and total must be different words.
cudaError_t launch_scan(const int32_t* lens, uint64_t* out_off, uint64_t* total, const uint64_t* carry_in, size_t n, cudaStream_t st);
// the gather alone: block i's max(lens[i], 0) bytes move from src + src_off[i] to dst + dst_off[i], one warp each
cudaError_t launch_gather(const uint8_t* src, const uint64_t* src_off, const int32_t* lens,
                          uint8_t* dst, const uint64_t* dst_off, size_t n, cudaStream_t st);

// ---- LZ4 Frame writer (frame_encode.cu, driven by compress_frames_dev in containers.cu for b200lz4f_compress_dev, and for
// b200lz4f_compress_host_hc on a device copy of its source).  flags: bit0 content checksum, bit1 block checksums, bit2
// content size.

// One call's descriptors, all device pointers.  An "item" is one block of a frame, or an empty frame (no block): the frame
// header rides on a frame's first item, the EndMark and content checksum on its last, so one scan of the item sizes places
// everything.  Items of a frame are consecutive; a frame's first / last item is where i_frame changes.
struct FramePlan {
    const uint8_t* src; uint8_t* dst; const uint8_t* slots;         // sources, the frames, one chunk's compressed blocks
    const uint64_t* b_soff; const int32_t* b_slen;                  // per block: source bytes
    const uint64_t* b_slot; const int32_t* b_clen;                  //   its slot in `slots` and the compressor's result
    uint64_t* b_poff; int32_t* b_plen; const uint32_t* b_sum;       //   the payload as written, and its XXH32 (flags bit 1)
    const uint32_t* i_frame; const int32_t* i_block;                // per item: frame, block (-1: an empty frame)
    int32_t* i_size; uint64_t* i_off;                               //   bytes it takes, where it starts in dst
    const uint64_t* f_len; const uint32_t* f_sum;                   // per frame: content size, content checksum (flags bit 0)
    uint64_t* f_off; uint64_t* f_end;                               //   where it starts and ends in dst
    uint32_t nitems; int bsCode; int flags;
    int level;                                                      // LZ4Block streams: the token's level nibble
};
// items [i0, i0 + n): their sizes (frame_size_kernel), and their block words and payloads (frame_emit_kernel, one warp each)
cudaError_t launch_frame_sizes(const FramePlan& p, uint32_t i0, uint32_t n, cudaStream_t st);
cudaError_t launch_frame_emit(const FramePlan& p, uint32_t i0, uint32_t n, cudaStream_t st);
// every item: headers, block checksums, EndMarks, content checksums, f_off / f_end (frame_seal_kernel)
cudaError_t launch_frame_seal(const FramePlan& p, cudaStream_t st);

// The incremental frame writer (b200lz4f_writer_*: writer_write_dev in containers.cu, kernels in frame_writer.cu).  One
// call is the frame writer's plan and chunk loop over the streams that write something: a "frame" of the plan is one such
// stream's part of the call (its blocks, or one item without a block), with the header only on the stream's first call
// (WRITER_HEAD) and the EndMark and content checksum only at its close (WRITER_TAIL).  Each stream's bytes go to its own
// range: item i of plan frame f lands at f_doff[f] + i_off[i] - i_off[f_first[f]].  p.f_len is the declared content size;
// f_off / f_end come back as the stream's range written.
enum { WRITER_HEAD = 1, WRITER_TAIL = 2 };
struct FrameWriterPlan {
    FramePlan p;
    const uint64_t* f_doff; const uint32_t* f_first; const uint8_t* f_mode;
};
// items [i0, i0 + n): their sizes, and their block words and payloads (one warp each)
cudaError_t launch_frame_writer_sizes(const FrameWriterPlan& w, uint32_t i0, uint32_t n, cudaStream_t st);
cudaError_t launch_frame_writer_emit(const FrameWriterPlan& w, uint32_t i0, uint32_t n, cudaStream_t st);
// every item: headers, block checksums, EndMarks, content checksums, f_off / f_end
cudaError_t launch_frame_writer_seal(const FrameWriterPlan& w, cudaStream_t st);
// A stream's state between calls, host data: its carried content checksum, whether its header is out, whether it is closed.
struct FrameWriterState { Xxh32Carry xxh; uint8_t head, done, pad[6]; };

// ---- LZ4 Frame reader: the container walk (LZ4FrameInputStream.nextFrameInfo / readHeader / readBlock as an index pass,
// LZ4FrameInputStream.java:132-321).  The host indexer (frame.cu) and the device one (frame_index.cu) both run walk_frames;
// only where the facts go differs (the Sink).
__host__ __device__ inline uint32_t rd32(const uint8_t* p) { return p[0] | (p[1] << 8) | (p[2] << 16) | ((uint32_t)p[3] << 24); }

// One frame as the walk found it.  At frame_begin: everything up to the header checksum byte; at frame_end: the rest.
struct WalkFrame {
    uint64_t desc_off, content_size, nblocks;
    uint32_t content_checksum;
    uint8_t flg, bd, hc_byte, desc_len;
    bool complete, has_checksum, has_size;   // read up to its EndMark (and content checksum); the content checks that apply
};
// Where it stopped and why; seen: any frame, skippable ones too.  A resumable walk (more input may come, or room is limited)
// may also stop in front of a unit: stop says why, at where that unit starts, need what it takes (see walk_frames_from).
struct WalkEnd { uint64_t ip; int err; bool seen, single_done; uint8_t stop; uint64_t at, need; };
enum { WALK_STOP_NONE = 0, WALK_STOP_INPUT = 1, WALK_STOP_ROOM = 2 };
// Where a walk starts, and where a resumable one stopped: between frames, inside a frame's blocks (that frame's FLG and BD),
// or inside a skippable frame's payload with `skip` bytes to go.  seen: any frame so far.  A fresh WalkPos is the start of
// a stream.
enum { WALK_AT_FRAME = 0, WALK_IN_BLOCKS = 1, WALK_IN_SKIP = 2 };
struct WalkPos { uint64_t skip; uint8_t where, flg, bd; bool seen; };

// Walks the frames of src[0, n) from ip, which must be where a frame (or a skippable frame) starts.  Stops at the first frame
// boundary at or past stop_at, at the end of src, at the first malformed spot (err, -1 -2 -4 -10) or, with `single`, behind
// the first non-skippable frame.  Bounds are checked against n, never stop_at.  Per frame the sink gets frame_begin, one
// block(src_off, word, checksum) per complete block, and frame_end -- also for a frame the container breaks off inside
// (complete = false).  Whether an error is the container's or the reader's is the caller's to say (it depends on what came
// before ip).
//
// walk_frames_from is the same walk, resumable (the incremental reader, frame_reader.cu).  It starts at `pos`, which it
// leaves where it stopped.  A unit is a frame header (magic to HC byte), a block (word, payload and block checksum), the
// EndMark with its content checksum, or a skippable frame's 8-byte header; a skippable frame's payload is taken in any
// portions.  With `more` (bytes past n may come) a unit that src holds only in part is not an error: the walk stops in front
// of it (WALK_STOP_INPUT, need = the unit's length once that is readable, else the bytes that make it readable).  A block
// whose slot room (frame_slot_room) is above `room` stops it in front of that block (WALK_STOP_ROOM, need = that room);
// `room` is debited by each block taken.  A frame the walk enters inside its blocks gets frame_begin with desc_len 0 (no
// header in src) and only flg and bd set.  With a fresh pos, `more` false and room above 4 MiB it is walk_frames exactly.
__host__ __device__ inline uint64_t frame_slot_room(uint32_t bs, uint32_t size, bool raw);
#ifdef __CUDACC__
#pragma nv_exec_check_disable
#endif
template <class Sink>
__host__ __device__ inline WalkEnd walk_frames_from(const uint8_t* src, uint64_t n, uint64_t ip, uint64_t stop_at, bool single,
                                                    WalkPos& pos, bool more, uint64_t room, Sink& sink)
{
    WalkEnd e{ ip, 0, pos.seen, false, WALK_STOP_NONE, ip, 0 };
    uint64_t unit = ip;                                                         // where the unit being read starts
    // src ends inside the unit at `unit`, which takes `len` bytes: more may come, or the stream is cut short
#define WALK_SHORT(len) do { if (more) { e.stop = WALK_STOP_INPUT; e.need = (len); ip = unit; } else e.err = -1; } while (0)
    bool in_blocks = pos.where == WALK_IN_BLOCKS;
    if (pos.where == WALK_IN_SKIP) {                                            // the rest of a skippable payload
        const uint64_t t = pos.skip < n - ip ? pos.skip : n - ip;
        ip += t; pos.skip -= t; unit = ip;
        if (pos.skip) { if (more) { e.stop = WALK_STOP_INPUT; e.need = pos.skip; } else e.err = -1; }
        else { pos.where = WALK_AT_FRAME; e.seen = true; }
    }
    while (!e.err && !e.stop && (in_blocks || (ip < n && ip < stop_at))) {
        WalkFrame f{};
        if (in_blocks) {                                                        // a frame the walk enters inside its blocks
            f.flg = pos.flg; f.bd = pos.bd; f.has_size = f.flg & 8; in_blocks = false; pos.where = WALK_AT_FRAME;
        } else {
            unit = ip;
            if (n - ip < 4) { WALK_SHORT(4); break; }
            const uint32_t magic = rd32(src + ip); ip += 4;
            if ((magic >> 4) == (0x184D2A50u >> 4)) {                           // skippable (:154,162-173)
                if (n - ip < 4) { WALK_SHORT(8); break; }
                const uint32_t sz = rd32(src + ip); ip += 4;
                if (n - ip < sz) {
                    if (!more) { e.err = -1; break; }
                    pos.where = WALK_IN_SKIP; pos.skip = sz - (n - ip); ip = unit = n;
                    e.stop = WALK_STOP_INPUT; e.need = pos.skip; break;
                }
                ip += sz; e.seen = true; continue;
            }
            if (magic != 0x184D2204u) { e.err = -2; break; }                    // (:151)
            f.desc_off = ip;
            if (n - ip < 3) { WALK_SHORT(n - ip ? 7 + ((src[ip] & 8) ? 8 : 0) : 5); break; }
            f.flg = src[ip++]; f.bd = src[ip++];
            if ((f.flg >> 6) != 1 || (f.flg & 2) || !(f.flg & 0x20) || (f.flg & 1)) { e.err = -10; break; }   // version, reserved, B.Indep, dictID
            if ((f.bd & 0x8F) || (f.bd >> 4) < 4) { e.err = -10; break; }
            f.has_size = f.flg & 8;
            if (f.has_size) { if (n - ip < 9) { WALK_SHORT(15); break; } f.content_size = (uint64_t)rd32(src + ip) | ((uint64_t)rd32(src + ip + 4) << 32); ip += 8; }
            if (n - ip < 1) { WALK_SHORT(7); break; }
            f.desc_len = (uint8_t)(ip - f.desc_off);
            f.hc_byte = src[ip++];
        }
        const uint32_t bs = 1u << (8 + 2 * (f.bd >> 4));
        sink.frame_begin(f);
        for (;;) {                                                              // readBlock (:258-321)
            unit = ip;
            if (n - ip < 4) { WALK_SHORT(4); break; }
            const uint32_t word = rd32(src + ip); ip += 4;
            const uint32_t sz = word & 0x7FFFFFFFu;
            if (sz == 0) break;                                                 // EndMark
            if (sz > bs) { e.err = -4; break; }
            const uint64_t at = ip, len = 4ull + sz + ((f.flg & 0x10) ? 4 : 0);
            if (n - ip < sz) { WALK_SHORT(len); break; }
            ip += sz;
            uint32_t sum = 0;
            if (f.flg & 0x10) { if (n - ip < 4) { WALK_SHORT(len); break; } sum = rd32(src + ip); ip += 4; }
            const uint64_t need = frame_slot_room(bs, sz, word >> 31);
            if (need > room) { e.stop = WALK_STOP_ROOM; e.need = need; ip = unit; break; }
            room -= need;
            sink.block(at, word, sum);
            f.nblocks++;
        }
        f.complete = !e.err && !e.stop;
        f.has_checksum = f.complete && (f.flg & 4);
        if (f.has_checksum) {
            if (n - ip < 4) { WALK_SHORT(8); f.complete = false; f.has_checksum = false; }
            else { f.content_checksum = rd32(src + ip); ip += 4; }
        }
        if (!f.complete) f.has_size = false;
        sink.frame_end(f); e.seen = true;
        if (e.stop) { pos.where = WALK_IN_BLOCKS; pos.flg = f.flg; pos.bd = f.bd; break; }
        if (single) { e.single_done = true; break; }                           // readSingleFrame (:83-91, 327, 346): the rest is not read
        if (e.err) break;
    }
#undef WALK_SHORT
    if (more && !e.err && !e.stop && !e.single_done && ip >= n) { e.stop = WALK_STOP_INPUT; e.need = 4; unit = ip; }
    pos.seen = e.seen;
    e.ip = ip;
    e.at = (e.err || e.stop) ? unit : ip;
    return e;
}

#ifdef __CUDACC__
#pragma nv_exec_check_disable
#endif
template <class Sink>
__host__ __device__ inline WalkEnd walk_frames(const uint8_t* src, uint64_t n, uint64_t ip, uint64_t stop_at, bool single, Sink& sink)
{
    WalkPos pos{};
    return walk_frames_from(src, n, ip, stop_at, single, pos, false, ~0ull, sink);
}

// The slot layout of the frame readers' decode (frame.cu's IndexSink, frame_streams.cu): a stored block needs its own size, a
// compressed one cannot decode to more than 255 bytes per byte (one length byte adds at most 255) -- so a stream of tiny
// flushed blocks asks for what it can fill, not for blockMaxSize each.  room is the decoder's capacity; a block takes
// frame_slot_bytes of the layout: full blocks exactly bs, so a frame without short blocks in the middle stays contiguous,
// the rest rounded up to 16.
__host__ __device__ inline uint64_t frame_slot_room(uint32_t bs, uint32_t size, bool raw)
{
    return raw ? size : (255ull * size < bs ? 255ull * size : bs);
}
__host__ __device__ inline uint64_t frame_slot_bytes(uint64_t room, uint32_t bs) { return room >= bs ? bs : ((room + 15) & ~15ull); }

// The device walk (frame_index.cu): one thread per segment [seg_start, seg_end) of the container, records into a region of
// its own.  A record is 16 bytes: a frame takes two (written at frame_end into the pair reserved at frame_begin), a block one;
// they come in stream order.  A walker whose region is full keeps counting (WalkSummary.nrec) but stops writing.
struct WalkSeg { uint64_t start, end, rec_off, rec_cap; };   // rec_off / rec_cap in records
struct WalkSummary { uint64_t ip, nrec; int32_t err; uint32_t flags; };
enum { WALK_SEEN = 1, WALK_SINGLE_DONE = 2 };
struct WalkRec { uint64_t a, b; };
// walkers [0, m): summaries, and lens[j] = the records walker j wrote (min(nrec, rec_cap))
cudaError_t launch_frame_walk(const uint8_t* src, uint64_t n, bool single, const WalkSeg* segs, WalkSummary* sum, int32_t* lens,
                              WalkRec* recs, uint32_t m, cudaStream_t st);
// walker j's lens[j] records move from recs + segs[j].rec_off to packed + pos[j]
cudaError_t launch_frame_pack(const WalkSeg* segs, const int32_t* lens, const uint64_t* pos, const WalkRec* recs, WalkRec* packed,
                              uint32_t m, cudaStream_t st);

// The device reader of many independent frame streams (frame_streams_decompress_dev in frame.cu, kernels in
// frame_streams.cu), all device pointers.  Per stream: its bytes and room, the counting walk's counts (FS_* rows of cnt, each
// ns entries, and their exclusive prefixes in pos), its tail code and end, and the results.  The records of every block and
// frame, in stream order, follow decode_dev's descriptor arrays (IndexLayout in frame.cu): c_* compressed blocks (BatchArgs of
// the safe decoder into the slots), r_* stored blocks (gather into the slots), k_* every block (the chained content checksum's
// view, and where the verdict puts it in d_dst: k_dst / k_len), b_* checksummed blocks, h_* frame descriptors, fr_* every
// frame, f_* frames with a content checksum.
enum { FS_COMP, FS_RAW, FS_BSUM, FS_FRAME, FS_FSUM, FS_SLOT16, FS_ROWS };     // counts per stream; slots in 16-byte units
struct FrameStreamRead {
    const uint8_t* src;
    const uint64_t *s_off, *s_len, *d_off, *d_cap;
    int32_t* cnt; const uint64_t* pos;                                  // cnt[row * ns + s], pos likewise
    int32_t* tail; uint64_t* ip; int32_t* over;                         // over: set when a stream's counts do not fit int32
    int64_t* result; uint64_t *consumed, *content;
    uint64_t *c_soff, *c_doff; int32_t *c_slen, *c_dcap, *c_res;
    uint64_t *r_soff, *r_doff; int32_t* r_len;
    int32_t *k_comp, *k_rawlen; uint64_t *k_off, *k_dst; int32_t* k_len;
    uint64_t* b_off; int32_t* b_len; uint32_t *b_want, *b_out;
    uint64_t* h_off; int32_t* h_len; uint32_t* h_out;
    uint32_t *fr_first, *fr_nblk; int32_t *fr_bsum, *fr_fsum; uint64_t* fr_size; uint32_t* fr_bits;   // bits: hc_byte, has_size
    uint32_t *f_first, *f_nblk, *f_want, *f_out;
    uint32_t ns; bool single;
};
// one thread per stream: with `record` false the counts, tail and ip; with it every record
cudaError_t launch_frame_streams_walk(const FrameStreamRead& r, bool record, cudaStream_t st);
// one warp per stream: result, consumed, content, and each block's k_dst / k_len (0 for a stream that fails)
cudaError_t launch_frame_streams_verdict(const FrameStreamRead& r, cudaStream_t st);

// The incremental reader (b200lz4f_reader_*: frame_reader_read_dev in frame.cu, kernels in frame_reader.cu).  A stream's
// state between calls, host data that goes up with a call's arguments and comes back with its results: where its walk is,
// the open frame's declared and counted content and its content checksum, and the latched status.
static constexpr int32_t READER_MORE_INPUT = 0, READER_MORE_ROOM = 1, READER_DONE = 2;
struct FrameReaderState {
    uint64_t skip, declared, counted;                   // WalkPos.skip; the open frame's content size (FLG bit 3), content so far
    Xxh32Carry xxh;                                     // the open frame's content checksum (FLG bit 2)
    int32_t status;                                     // 0 while reading; READER_DONE or -1 .. -10 once latched
    uint8_t where, flg, bd, seen;                       // WalkPos
};
// One call, all device pointers.  r holds the per-stream arguments and decode_dev's descriptor arrays as for
// b200lz4f_decompress_streams_dev (r.consumed is src_consumed; r.result, r.content are unused).  Per block its unit's start in
// the piece (k_at); per frame the part of it in this call (fr_mode READER_FR_*, where its header unit and its EndMark unit
// start); per content-checksummed frame the carried checksum (f_carry, f_mode XXH_CARRY_*).
enum { READER_FR_HEAD = 1, READER_FR_END = 2 };
struct FrameReaderRead {
    FrameStreamRead r;
    const uint8_t* eof;
    const FrameReaderState* st_in; FrameReaderState* st_out;
    int32_t* status; uint64_t *produced, *need;
    uint64_t* k_at;
    uint64_t *fr_at, *fr_end_at; uint32_t* fr_mode;
    Xxh32Carry* f_carry; uint8_t* f_mode;
};
// one thread per stream: with `record` false the counts (FS_* rows of r.cnt), the walk's end in tail / consumed / need /
// st_out; with it every record
cudaError_t launch_frame_reader_walk(const FrameReaderRead& q, bool record, cudaStream_t st);
// one warp per stream: status, consumed, produced, need, st_out, and each block's k_dst / k_len (0 from the first failing unit)
cudaError_t launch_frame_reader_verdict(const FrameReaderRead& q, cudaStream_t st);

// ---- "LZ4Block" streams (LZ4BlockOutputStream.java:203-266, LZ4BlockInputStream.java:191-264).  The writer is the frame
// writer's loop (compress_blocks_dev in containers.cu) with lz4block.cu's item sizes, emit and seal: the same FramePlan, a
// "frame" being one stream, its last item carrying the empty end block.
static constexpr int LZ4BLOCK_HEADER = 8 + 1 + 4 + 4 + 4;          // magic, token, compressed and original length, checksum
static constexpr int LZ4BLOCK_RAW = 0x10, LZ4BLOCK_LZ4 = 0x20;     // the token's method nibble
static constexpr uint32_t LZ4BLOCK_SEED = 0x9747b28cu;             // LZ4BlockOutputStream.java:56
static constexpr uint32_t LZ4BLOCK_MAGIC_LO = 0x42345A4Cu, LZ4BLOCK_MAGIC_HI = 0x6B636F6Cu;   // "LZ4Block", little endian
cudaError_t launch_lz4block_sizes(const FramePlan& p, uint32_t i0, uint32_t n, cudaStream_t st);
cudaError_t launch_lz4block_emit(const FramePlan& p, uint32_t i0, uint32_t n, cudaStream_t st);
// every item: block checksums (b_sum, masked to 28 bits), end blocks, f_off / f_end
cudaError_t launch_lz4block_seal(const FramePlan& p, cudaStream_t st);
// The incremental LZ4Block writer (b200lz4block_writer_*: writer_write_dev in containers.cu, as for frames): the incremental
// frame writer's plan (FrameWriterPlan) with lz4block.cu's writer kernels.  No header is ever due; WRITER_TAIL puts the end
// block on the plan frame's last item.  p.f_len is not read.
cudaError_t launch_lz4block_writer_sizes(const FrameWriterPlan& w, uint32_t i0, uint32_t n, cudaStream_t st);
cudaError_t launch_lz4block_writer_emit(const FrameWriterPlan& w, uint32_t i0, uint32_t n, cudaStream_t st);
// every item: block checksums, end blocks, f_off / f_end as the stream's range written
cudaError_t launch_lz4block_writer_seal(const FrameWriterPlan& w, cudaStream_t st);

// The reader's walk of one stream, src[0, n), LZ4BlockInputStream.refill's header rules (:191-264).  Per block whose payload
// is complete the sink gets block(payload offset, raw, compressed length, original length, checksum).  Returns where the walk
// stopped and why: err 0 at the end of the stream (the first empty block with `stop`; without it, the end of src, quietly also
// inside a header, :193-194), -1 premature end, -2 "Stream is corrupted".  Capacity is not the walk's: see Lz4BlockRoom.
//
// walk_lz4block_from is the same walk, resumable (the incremental reader, lz4block.cu).  A unit is a 21-byte header with its
// payload.  With `more` (bytes past n may come) a unit that src holds only in part is not an error: the walk stops in front
// of it (stop WALK_STOP_INPUT, need = the unit's length once its header is readable, else 21).  A block whose original length
// is above `room` stops it in front of that block (WALK_STOP_ROOM, need = that length); `room` is debited by each block
// taken.  On an error ip is where the failing unit starts.  With `more` false and room ~0 it is walk_lz4block exactly.
// walk_lz4block is the same code with Resumable false, so the whole-stream readers carry no room or input bookkeeping.
struct Lz4BlockEnd { uint64_t ip; int err; uint8_t stop = WALK_STOP_NONE; uint64_t need = 0; };
#ifdef __CUDACC__
#pragma nv_exec_check_disable
#endif
template <bool Resumable, class Sink>
__host__ __device__ inline Lz4BlockEnd walk_lz4block_impl(const uint8_t* src, uint64_t n, bool stop, bool more, uint64_t room, Sink& sink)
{
    uint64_t ip = 0;
    for (;;) {
        if (n - ip < (uint64_t)LZ4BLOCK_HEADER) {
            if (Resumable && more) return { ip, 0, WALK_STOP_INPUT, (uint64_t)LZ4BLOCK_HEADER };
            return stop ? Lz4BlockEnd{ ip, -1 } : Lz4BlockEnd{ n, 0 };
        }
        const uint8_t* h = src + ip;
        if (rd32(h) != LZ4BLOCK_MAGIC_LO || rd32(h + 4) != LZ4BLOCK_MAGIC_HI) return { ip, -2 };
        const int token = h[8], method = token & 0xF0, level = 10 + (token & 0x0F);
        if (method != LZ4BLOCK_RAW && method != LZ4BLOCK_LZ4) return { ip, -2 };
        const int32_t clen = (int32_t)rd32(h + 9), olen = (int32_t)rd32(h + 13);
        const uint32_t check = rd32(h + 17);
        if (olen > (1 << level) || olen < 0 || clen < 0 || (olen == 0 && clen != 0) || (olen != 0 && clen == 0) ||
            (method == LZ4BLOCK_RAW && olen != clen)) return { ip, -2 };
        const uint64_t unit = ip;
        ip += LZ4BLOCK_HEADER;
        if (olen == 0) {                                                        // empty block (:225-233)
            if (check != 0) return { Resumable ? unit : ip, -2 };
            if (stop) return { ip, 0 };
            continue;
        }
        if (n - ip < (uint64_t)clen) {
            if (Resumable && more) return { unit, 0, WALK_STOP_INPUT, LZ4BLOCK_HEADER + (uint64_t)clen };
            return { Resumable ? unit : ip, -1 };
        }
        if (Resumable) {
            if ((uint64_t)olen > room) return { unit, 0, WALK_STOP_ROOM, (uint64_t)olen };
            room -= (uint64_t)olen;
        }
        sink.block(ip, method == LZ4BLOCK_RAW, clen, olen, check);
        ip += (uint64_t)clen;
    }
}
#ifdef __CUDACC__
#pragma nv_exec_check_disable
#endif
template <class Sink>
__host__ __device__ inline Lz4BlockEnd walk_lz4block_from(const uint8_t* src, uint64_t n, bool stop, bool more, uint64_t room, Sink& sink)
{
    return walk_lz4block_impl<true>(src, n, stop, more, room, sink);
}
#ifdef __CUDACC__
#pragma nv_exec_check_disable
#endif
template <class Sink>
__host__ __device__ inline Lz4BlockEnd walk_lz4block(const uint8_t* src, uint64_t n, bool stop, Sink& sink)
{
    return walk_lz4block_impl<false>(src, n, stop, false, ~0ull, sink);
}
// dst_cap applied behind the walk, the same way by both readers: blocks are taken while the prefix sum of their original
// lengths fits; the first one that does not is the stream's -9 (unless a block before it fails its decode or checksum: -2).
struct Lz4BlockRoom {
    uint64_t cap, used = 0; bool full = false;
    __host__ __device__ bool take(int32_t olen)
    {
        if (full || cap - used < (uint64_t)olen) { full = true; return false; }
        used += (uint64_t)olen;
        return true;
    }
};

// The device reader (lz4block_decompress_dev in containers.cu), all device pointers.  Per stream: its bytes and room, what the
// counting walk found, where its records go (exclusive prefixes of the counts) and the results.  Per block that fits, in
// stream order: b_*; per compressed block c_*, per stored block r_* (BatchArgs of the fast decoder and of the gather).
struct Lz4BlockRead {
    const uint8_t* src;
    const uint64_t *s_off, *s_len, *d_off, *d_cap;
    int32_t *n_comp, *n_raw, *tail; uint64_t *ip, *content;             // the counting walk (tail: -9 when a block does not fit)
    const uint64_t *p_comp, *p_raw;
    int64_t* result; uint64_t* consumed;
    uint64_t *c_soff, *c_doff; int32_t *c_clen, *c_olen, *c_res;
    uint64_t *r_soff, *r_doff; int32_t* r_len;
    uint64_t* b_doff; int32_t *b_len, *b_comp; uint32_t *b_want, *b_sum;
    uint32_t ns; bool stop;
};
// one thread per stream: with `record` false the counts, tail, ip and content; with it the records of the blocks that fit
cudaError_t launch_lz4block_walk(const Lz4BlockRead& r, bool record, cudaStream_t st);
// one warp per stream: result, consumed
cudaError_t launch_lz4block_verdict(const Lz4BlockRead& r, cudaStream_t st);

// The incremental reader (b200lz4block_reader_*: lz4block_reader_read_dev in containers.cu, kernels in lz4block.cu), all
// device pointers.  r holds the per-stream arguments and the block records as for b200lz4block_decompress_dev (r.consumed
// is src_consumed; r.ip, r.content and r.result are unused).  Per stream its latched status (st_in: 0 while reading), the
// results, and per block where its unit starts in the piece (k_at).
struct Lz4BlockReaderRead {
    Lz4BlockRead r;
    const uint8_t* eof; const int32_t* st_in;
    int32_t* status; uint64_t *produced, *need;
    uint64_t* k_at;
};
// one thread per stream: with `record` false the counts, the walk's end in tail / consumed / need; with it every record
cudaError_t launch_lz4block_reader_walk(const Lz4BlockReaderRead& q, bool record, cudaStream_t st);
// one warp per stream: status, consumed, produced, need, cut at the first block that fails its decode or checksum
cudaError_t launch_lz4block_reader_verdict(const Lz4BlockReaderRead& q, cudaStream_t st);

// ---- length-prefixed records (LZ4CompressorWithLength / LZ4DecompressorWithLength).  The writer is the frame writer's loop
// (compress_blocks_dev) with with_length.cu's item sizes and emit: a "frame" is one record, one item and one block of its
// whole length (an empty record too).  The emit also writes f_off / f_end, so there is no seal.
cudaError_t launch_with_length_sizes(const FramePlan& p, uint32_t i0, uint32_t n, cudaStream_t st);
cudaError_t launch_with_length_emit(const FramePlan& p, uint32_t i0, uint32_t n, cudaStream_t st);

// The device reader (with_length_decompress_dev in containers.cu), all device pointers.  Per record: its bytes and room, the
// decoder's arguments (BatchArgs of the fast or safe decoder, dst_off being d_off), the header's verdict and the results.
struct WithLengthRead {
    const uint8_t* src;
    const uint64_t *s_off, *s_len, *d_cap;
    uint64_t* b_soff; int32_t *b_slen, *b_dlen, *b_res;
    int32_t* head;                                                      // 0, or -1 when the header rejects the record
    int64_t *result, *orig_len;
    uint32_t n; bool safe;
};
// one thread per record: head, orig_len and the decoder's arguments
cudaError_t launch_with_length_head(const WithLengthRead& r, cudaStream_t st);
// one thread per record: result
cudaError_t launch_with_length_verdict(const WithLengthRead& r, cudaStream_t st);

// Average buffer length from which the hash batches give each buffer a whole warp (launch_xxh*_long) instead of a lane.
static constexpr uint64_t XXH_LONG_AVG = 32768;

// LZ4_compressBound(len) (lz4.h:212) without its range check, and the room one block takes in a packed compress
// staging area: that bound rounded up to 16 bytes.
static inline uint64_t compress_bound(uint64_t len) { return len + len / 255 + 16; }
static inline uint64_t aligned_compress_bound(uint64_t len) { return (compress_bound(len) + 15) & ~uint64_t(15); }

extern std::atomic<unsigned long long> g_launch_count;      // every kernel launch the library makes (any thread): b200lz4_launch_count()
// one launch's result, the launch counted
static inline cudaError_t counted(cudaError_t e) { g_launch_count.fetch_add(1, std::memory_order_relaxed); return e; }

// ---- host layer shared by capi.cu, containers.cu and frame.cu
extern const size_t CHUNK_SPAN;                            // bytes of source per chunk of a chunked call (B200LZ4_CHUNK_MB, default 256)
static constexpr size_t CHUNK_BLOCKS = 1 << 16;            // blocks per chunk at most
int fail_arg(const char* what);                            // set the thread's error message, return B200LZ4_E_ARG
int fail_cuda(cudaError_t e, const char* where);           // ... B200LZ4_E_CUDA or _NODEVICE
// The ranges of a device call over ns streams (or records): every src_len[k] at most src_max, every dst_cap[k] at most 2^47,
// no dst_off[k] + dst_cap[k] past 2^64, and d_src / d_dst not NULL when the streams have bytes / room.  0 with the summed
// lengths and capacities in bytes and room, or B200LZ4_E_ARG.
int check_stream_ranges(size_t ns, const uint64_t* src_len, uint64_t src_max, const uint64_t* dst_off, const uint64_t* dst_cap,
                        const void* d_src, const void* d_dst, uint64_t& bytes, uint64_t& room);
// a failed CUDA call: the thread's error message names it, the caller returns fail_cuda's code
#define CK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) return b200::fail_cuda(e_, #call); } while (0)
int reserve_device(uint8_t*& p, size_t& cap, size_t need, int slack_shift = 2);   // grow-or-keep device buffer
int reserve_pinned(uint8_t*& p, size_t& cap, size_t need);                       // grow-or-keep pinned buffer
// A call that fails half way waits for what it queued on its streams: the scratch it used stays the thread's, and the next
// call may reuse or free it.  Set done once the call has synchronised.
struct Drain {
    cudaStream_t a, b = nullptr; bool done = false;
    ~Drain() { if (!done) { cudaStreamSynchronize(a); if (b) cudaStreamSynchronize(b); } }
};
// The frame calls' second stream, one per thread and device: the writer's content checksums and the reader's chained content
// checksums run on it beside the caller's stream, from `fork` on, and every call joins it (`join`) before it returns.
struct SideStream { cudaStream_t st = nullptr; cudaEvent_t fork = nullptr, join = nullptr; };
// Grow-or-keep scratch of the frame writer, one per thread and device (it lives in the thread's context).
struct FrameScratch {
    uint8_t* d_plan = nullptr; size_t plan_cap = 0;        // the call's descriptors (FramePlan)
    uint8_t* h_plan = nullptr; size_t h_plan_cap = 0;      // pinned: their upload, and the results coming back
    uint8_t* d_slots = nullptr; size_t slots_cap = 0;      // one chunk's compressed blocks, bound-sized slots
    uint8_t* d_stage = nullptr; size_t stage_cap = 0;      // b200lz4f_compress_host_hc: the source at its 16-byte phase, then the frame
};
// Grow-or-keep scratch of the frame reader, same lifetime.  d_seg / h_seg serve every step in turn: the device walk, then
// decode_dev's descriptors and results, then the packing descriptors.
struct FrameReadScratch {
    uint8_t* d_seg = nullptr; size_t seg_cap = 0;          // walk: segments, summaries, counts, positions; decode: descriptors
    uint8_t* h_seg = nullptr; size_t h_seg_cap = 0;        // pinned: their upload, and what comes back
    uint8_t* d_recs = nullptr; size_t recs_cap = 0;        // the walkers' record regions
    uint8_t* d_packed = nullptr; size_t packed_cap = 0;    // the records, packed for one copy back
    uint8_t* d_slots = nullptr; size_t slots_cap = 0;      // decompress_dev: the decoded blocks, slot_bytes
};
// Both select the thread's device, like every entry point.  side (may be NULL): the side stream, created at its first use.
// idle (may be NULL): a stream of the thread's context that no call keeps busy between calls.
int get_frame_scratch(FrameScratch** out, SideStream** side = nullptr, cudaStream_t* idle = nullptr);
int get_frame_read_scratch(FrameReadScratch** out, SideStream** side = nullptr, cudaStream_t* idle = nullptr);

} // namespace b200
