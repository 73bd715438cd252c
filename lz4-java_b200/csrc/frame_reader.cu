// frame_reader.cu — the device half of the incremental frame reader (b200lz4f_reader_read_dev: frame_reader_read_dev in
// frame.cu).  Each of ns streams is one LZ4FrameInputStream(in, readSingleFrame) whose bytes arrive in pieces; a call takes
// the complete units at the start of each stream's piece, and the stream's state (FrameReaderState, kernels.h) carries the
// rest to the next call.  Every per-block and per-frame fact stays on the device:
//   frame_reader_walk_kernel     one thread per stream resumes the container walk (walk_frames_from, kernels.h, the other
//                                readers' walk too) from the carried state: first counting what it takes, then, behind scans
//                                of the counts, writing decode_dev's descriptor arrays, with the carried content checksum of
//                                a frame that began in an earlier call
//   (decode_dev's payload launches, the chained content checksum leaving the state of a frame that goes on in a later call)
//   frame_reader_verdict_kernel  one warp per stream: decode_dev's stream-order checks, cut at the first failing unit; the
//                                blocks in front of the cut go to d_dst, and the stream's new state, status and counts come out
// and one gather packs the blocks in front of each cut.
#include "common.cuh"
#include "kernels.h"

namespace b200 {

// The counting walk's sink: per stream the FS_* counts, as frame_streams.cu counts them, except that every frame with a
// content checksum gets a chained record (a frame that stops inside the call leaves its state there).
struct FrameReaderCountSink {
    uint64_t n[FS_ROWS] = {}; uint32_t bs = 0; uint8_t flg = 0;
    __device__ void frame_begin(const WalkFrame& w) { flg = w.flg; bs = 1u << (8 + 2 * (w.bd >> 4)); }
    __device__ void block(uint64_t, uint32_t word, uint32_t)
    {
        const uint32_t size = word & 0x7FFFFFFFu; const bool raw = word >> 31;
        n[raw ? FS_RAW : FS_COMP]++;
        if (flg & 0x10) n[FS_BSUM]++;
        n[FS_SLOT16] += frame_slot_bytes(frame_slot_room(bs, size, raw), bs) >> 4;
    }
    __device__ void frame_end(const WalkFrame&) { n[FS_FRAME]++; if (flg & 4) n[FS_FSUM]++; }
};

// The recording walk's sink: frame_streams.cu's records, plus where each unit starts in the piece (the cut's src_consumed)
// and which parts of each frame the call holds.  c, q, b, k, f, j: the stream's next compressed, stored, any and checksummed
// block, its next frame and content-checksummed frame; slot: the next slot byte; end: where the last unit taken ends.
struct FrameReaderRecordSink {
    const FrameReaderRead& q; const FrameReaderState& st; uint64_t soff, c, qr, b, k, f, j, slot;
    uint64_t first = 0, end = 0; int32_t bsum0 = -1; uint32_t bs = 0; uint8_t flg = 0; bool head = false;
    __device__ void frame_begin(const WalkFrame& w)
    {
        flg = w.flg; bs = 1u << (8 + 2 * (w.bd >> 4));
        first = b; bsum0 = (flg & 0x10) ? (int32_t)k : -1;
        head = w.desc_len != 0;
        end = head ? w.desc_off + w.desc_len + 1 : 0;
    }
    __device__ void block(uint64_t at, uint32_t word, uint32_t checksum)
    {
        const FrameStreamRead& r = q.r;
        const uint32_t size = word & 0x7FFFFFFFu; const bool raw = word >> 31;
        const uint64_t room = frame_slot_room(bs, size, raw);
        r.k_off[b] = slot; q.k_at[b] = at - 4;
        if (raw) {
            r.k_comp[b] = -1; r.k_rawlen[b] = (int32_t)size;
            r.r_soff[qr] = soff + at; r.r_doff[qr] = slot; r.r_len[qr++] = (int32_t)size;
        } else {
            r.k_comp[b] = (int32_t)c; r.k_rawlen[b] = 0;
            r.c_soff[c] = soff + at; r.c_doff[c] = slot; r.c_slen[c] = (int32_t)size; r.c_dcap[c++] = (int32_t)room;
        }
        if (flg & 0x10) { r.b_off[k] = soff + at; r.b_len[k] = (int32_t)size; r.b_want[k++] = checksum; }
        slot += frame_slot_bytes(room, bs);
        end = at + size + ((flg & 0x10) ? 4 : 0);
        b++;
    }
    __device__ void frame_end(const WalkFrame& w)
    {
        const FrameStreamRead& r = q.r;
        r.h_off[f] = soff + w.desc_off; r.h_len[f] = w.desc_len;
        r.fr_first[f] = (uint32_t)first; r.fr_nblk[f] = (uint32_t)(b - first); r.fr_bsum[f] = bsum0;
        r.fr_size[f] = w.content_size; r.fr_bits[f] = (uint32_t)w.hc_byte | ((flg & 8) ? 0x100u : 0u);
        q.fr_mode[f] = (head ? READER_FR_HEAD : 0u) | (w.complete ? READER_FR_END : 0u);
        q.fr_at[f] = head ? w.desc_off - 4 : 0; q.fr_end_at[f] = end;
        r.fr_fsum[f] = -1;
        if (flg & 4) {
            r.f_first[j] = (uint32_t)first; r.f_nblk[j] = (uint32_t)(b - first); r.f_want[j] = w.content_checksum;
            q.f_mode[j] = (uint8_t)((head ? 0 : XXH_CARRY_IN) | (w.complete ? 0 : XXH_CARRY_OUT));
            if (!head) q.f_carry[j] = st.xxh;
            r.fr_fsum[f] = (int32_t)j++;
        }
        f++;
    }
};

__global__ void __launch_bounds__(128)
frame_reader_walk_kernel(const FrameReaderRead q, bool record)
{
    const FrameStreamRead& r = q.r;
    const uint32_t s = blockIdx.x * 128 + threadIdx.x;
    if (s >= r.ns) return;
    const FrameReaderState st = q.st_in[s];
    const uint8_t* src = r.src + r.s_off[s];
    const uint64_t n = r.s_len[s];
    WalkPos pos{ st.skip, st.where, st.flg, st.bd, st.seen != 0 };
    const bool more = !q.eof[s];
    if (!record) {
        FrameReaderCountSink sink;
        FrameReaderState out = st;
        if (st.status) {                                                    // latched: nothing is read
            for (int row = 0; row < FS_ROWS; row++) r.cnt[(size_t)row * r.ns + s] = 0;
            r.tail[s] = st.status; r.consumed[s] = 0; q.need[s] = 0; q.st_out[s] = out;
            return;
        }
        const WalkEnd e = walk_frames_from(src, n, 0, n, r.single, pos, more, r.d_cap[s], sink);
        bool over = false;
        for (int row = 0; row < FS_ROWS; row++) {
            const uint64_t v = sink.n[row];
            over |= v > 0x7FFFFFFFull;
            r.cnt[(size_t)row * r.ns + s] = (int32_t)(v > 0x7FFFFFFFull ? 0x7FFFFFFFull : v);
        }
        if (over) *r.over = 1;
        // the walk's own end: its error, DONE behind the single frame or at the end of the stream (no frame at all, skippable
        // ones included, is -1 as for the host reader), or what it waits for
        r.tail[s] = e.err ? e.err : e.single_done ? READER_DONE
                  : e.stop == WALK_STOP_INPUT ? READER_MORE_INPUT : e.stop == WALK_STOP_ROOM ? READER_MORE_ROOM
                  : e.seen ? READER_DONE : -1;
        r.consumed[s] = e.at; q.need[s] = e.stop ? e.need : 0;
        out.skip = pos.skip; out.where = pos.where; out.flg = pos.flg; out.bd = pos.bd; out.seen = pos.seen;
        q.st_out[s] = out;
        return;
    }
    if (st.status) return;
    auto at = [&](int row) { return r.pos[(size_t)row * r.ns + s]; };
    FrameReaderRecordSink sink{ q, st, r.s_off[s], at(FS_COMP), at(FS_RAW), at(FS_COMP) + at(FS_RAW), at(FS_BSUM), at(FS_FRAME),
                                at(FS_FSUM), at(FS_SLOT16) << 4 };
    walk_frames_from(src, n, 0, n, r.single, pos, more, r.d_cap[s], sink);
}

// decode_dev's verdict for one stream per warp, 32 blocks at a time, cut at the first failing unit: frame by frame the
// descriptor hash (-3) of a header in this call, block by block its checksum (-5) and its decode (-6), at an EndMark in this
// call the content checksum (-7) and size (-8) over the frame's whole content (what earlier calls counted and hashed
// included); then the walk's own end.  The blocks in front of the cut are placed back to back from dst_off; a frame still
// open at the end hands its counted content and checksum state to the stream's new state.
__global__ void __launch_bounds__(128)
frame_reader_verdict_kernel(const FrameReaderRead q)
{
    const FrameStreamRead& r = q.r;
    const uint32_t s = blockIdx.x * 4 + (threadIdx.x >> 5);
    if (s >= r.ns) return;
    const int lane = lane_id();
    const size_t ns = r.ns;
    const FrameReaderState& st = q.st_in[s];
    if (st.status) {
        if (lane == 0) { q.status[s] = st.status; q.produced[s] = 0; }
        return;
    }
    const uint64_t f0 = r.pos[FS_FRAME * ns + s], f1 = f0 + (uint64_t)r.cnt[FS_FRAME * ns + s];
    const uint64_t b0 = r.pos[FS_COMP * ns + s] + r.pos[FS_RAW * ns + s];
    const uint64_t b1 = b0 + (uint64_t)r.cnt[FS_COMP * ns + s] + (uint64_t)r.cnt[FS_RAW * ns + s];
    int32_t bad = 0;
    uint64_t cut = b1, cut_at = 0, produced = 0, open_count = 0, open_size = 0;
    int32_t open_fs = -1;
    for (uint64_t f = f0; f < f1; f++) {
        const uint32_t bits = r.fr_bits[f], mode = q.fr_mode[f];
        const uint32_t first = r.fr_first[f], nblk = r.fr_nblk[f];
        if ((mode & READER_FR_HEAD) && ((r.h_out[f] >> 8) & 0xFF) != (bits & 0xFF)) { bad = -3; cut = first; cut_at = q.fr_at[f]; break; }
        const int32_t bsum0 = r.fr_bsum[f];
        uint64_t len = 0;
        for (uint32_t base = 0; base < nblk; base += 32) {
            const uint32_t k = base + (uint32_t)lane;
            int32_t e = 0, l = 0;
            if (k < nblk) {
                const uint32_t b = first + k;
                if (bsum0 >= 0 && r.b_out[bsum0 + k] != r.b_want[bsum0 + k]) e = -5;
                else {
                    const int32_t c = r.k_comp[b];
                    l = c < 0 ? r.k_rawlen[b] : r.c_res[c];
                    if (l < 0) { e = -6; l = 0; }
                }
            }
            const uint32_t m = __ballot_sync(B200_FULL, e != 0);
            const int at = m ? __ffs((int)m) - 1 : 32;
            if (lane >= at) l = 0;                                          // the blocks in front of the first failing one
            for (int d = 16; d; d >>= 1) l += __shfl_xor_sync(B200_FULL, l, d);
            len += (uint64_t)l;
            if (m) { bad = __shfl_sync(B200_FULL, e, at); cut = first + base + (uint32_t)at; cut_at = q.k_at[cut]; break; }
        }
        produced += len;
        if (bad) break;
        const bool head = mode & READER_FR_HEAD;
        const uint64_t count = (head ? 0 : st.counted) + len, size = head ? r.fr_size[f] : st.declared;
        if (mode & READER_FR_END) {
            const int32_t fs = r.fr_fsum[f];
            if (fs >= 0 && r.f_out[fs] != r.f_want[fs]) bad = -7;
            else if ((bits & 0x100) && size != count) bad = -8;
            if (bad) { cut = first + nblk; cut_at = q.fr_end_at[f]; break; }
        } else {
            open_count = count; open_size = size; open_fs = r.fr_fsum[f];
        }
    }
    const int32_t status = bad ? bad : r.tail[s];
    if (lane == 0) {
        FrameReaderState& out = q.st_out[s];                               // the walk's position is already there
        q.status[s] = status; q.produced[s] = produced;
        if (bad) r.consumed[s] = cut_at;
        if (status < 0 || status == READER_DONE) { q.need[s] = 0; out.status = status; }
        else {
            out.counted = open_count; out.declared = open_size;
            if (open_fs >= 0) out.xxh = q.f_carry[open_fs];
        }
    }
    uint64_t run = r.d_off[s];
    for (uint64_t base = b0; base < b1; base += 32) {
        const uint64_t b = base + (uint64_t)lane;
        int32_t l = 0;
        if (b < cut) { const int32_t c = r.k_comp[b]; l = c < 0 ? r.k_rawlen[b] : r.c_res[c]; }
        int32_t x = l;                                                      // inclusive prefix over the lanes
        for (int d = 1; d < 32; d <<= 1) { const int32_t y = __shfl_up_sync(B200_FULL, x, d); if (lane >= d) x += y; }
        if (b < b1) { r.k_dst[b] = run + (uint64_t)(x - l); r.k_len[b] = l; }
        run += (uint64_t)__shfl_sync(B200_FULL, x, 31);
    }
}

// launchers: the same code in the emulator build (B200_LAUNCH)
cudaError_t launch_frame_reader_walk(const FrameReaderRead& q, bool record, cudaStream_t st)
{
    if (q.r.ns == 0) return cudaSuccess;
    B200_LAUNCH(frame_reader_walk_kernel, (q.r.ns + 127) / 128, 128, st, q, record);
    return cudaGetLastError();
}
cudaError_t launch_frame_reader_verdict(const FrameReaderRead& q, cudaStream_t st)
{
    if (q.r.ns == 0) return cudaSuccess;
    B200_LAUNCH(frame_reader_verdict_kernel, (q.r.ns + 3) / 4, 128, st, q);
    return cudaGetLastError();
}

} // namespace b200
