/*
 * b200lz4.h — C ABI of libb200lz4.so, the H100 (sm_90a) LZ4 block codec + XXHash backend ("B200" is its name).
 *
 * This is the drop-in boundary for the one hot path of lz4-java: the functions below are
 * what a `net.jpountz.lz4.LZ4B200JNI` / `net.jpountz.xxhash.XXHashB200JNI` shim binds, in
 * the same way the reference's JNI shim binds the vendored C:
 *
 *   reference call site (under /root/reference)                       replaced by
 *   src/jni/net_jpountz_lz4_LZ4JNI.c:75   LZ4_compress_default        b200lz4_compress_default
 *   src/jni/net_jpountz_lz4_LZ4JNI.c:122  LZ4_compress_HC             b200lz4_compress_HC
 *   src/jni/net_jpountz_lz4_LZ4JNI.c:169  LZ4_decompress_fast         b200lz4_decompress_fast_bounded
 *   src/jni/net_jpountz_lz4_LZ4JNI.c:216  LZ4_decompress_safe         b200lz4_decompress_safe
 *   src/jni/net_jpountz_lz4_LZ4JNI.c:237  LZ4_compressBound           b200lz4_compressBound
 *   src/jni/net_jpountz_xxhash_XXHashJNI.c:54,78    XXH32             b200xxh32
 *   src/jni/net_jpountz_xxhash_XXHashJNI.c:164,188  XXH64             b200xxh64
 *   src/jni/net_jpountz_xxhash_XXHashJNI.c:89-145   XXH32_* state     b200xxh32_create/reset/update/digest/free
 *   src/jni/net_jpountz_xxhash_XXHashJNI.c:199-255  XXH64_* state     b200xxh64_create/reset/update/digest/free
 *
 * All arithmetic runs in hand-written CUDA kernels; there is NO CPU fallback: every entry
 * point returns B200LZ4_E_NODEVICE (or 0 for the hash one-shots, with b200lz4_last_error()
 * set) when no sm_90 device/driver is usable.
 *
 * Return conventions are the reference's (SURVEY.md §8b):
 *   compress          > 0 compressed size, 0 if dst is too small / input too large
 *   decompress_safe   >= 0 decoded size, < 0 == -(error position)-1   (lz4.c:2337)
 *   decompress_fast   >= 0 compressed bytes consumed, -1 on any error  (lz4.c:1890)
 *
 * Besides the one-block-per-call functions (what the net.jpountz API needs, n = 1), the
 * library exposes BATCH calls: one launch over n independent blocks.  These are the calls
 * that make a GPU backend meaningful (SURVEY.md §7 "hard parts" 1); the single-block calls
 * are the n = 1 case of the host batch path.
 */
#ifndef B200LZ4_H
#define B200LZ4_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200LZ4_VERSION        100          /* 0.1.0 */
#define B200LZ4_E_NODEVICE     (-2147483647)       /* INT_MIN + 1: no usable CUDA device / driver            */
#define B200LZ4_E_CUDA         (-2147483646)       /* INT_MIN + 2: CUDA runtime error, see b200lz4_last_error */
#define B200LZ4_E_ARG          (-2147483645)       /* INT_MIN + 3: invalid argument                           */

/* ---------------------------------------------------------------- library / device */
int         b200lz4_version(void);
int         b200lz4_device_count(void);           /* >= 0, or B200LZ4_E_NODEVICE            */
int         b200lz4_set_device(int device);       /* device used by the calling thread      */
const char* b200lz4_last_error(void);             /* thread-local, never NULL                */
/* The hash entry points return the hash VALUE (like XXH32/XXH64, xxhash.c:392,855), so they cannot return an error
 * code: b200xxh32 / b200xxh64 / b200xxh*_digest clear this thread-local status on entry and leave a B200LZ4_E_* in it
 * when they could not compute (they then return 0).  A binding must check it after each of those calls and throw. */
int         b200lz4_last_status(void);
/* Pin / unpin a caller-owned host range (e.g. a Java DirectByteBuffer) so the host batch
 * calls DMA straight from/to it.  Optional: unpinned memory works, slower. */
int         b200lz4_host_register(void* p, size_t bytes);
int         b200lz4_host_unregister(void* p);

/* ---------------------------------------------------------------- one block per call, HOST buffers */
int b200lz4_compressBound(int inputSize);                                            /* lz4.h:212 */
int b200lz4_compress_default(const char* src, char* dst, int srcSize, int dstCapacity);
int b200lz4_compress_HC(const char* src, char* dst, int srcSize, int dstCapacity, int level);
int b200lz4_decompress_safe(const char* src, char* dst, int compressedSize, int dstCapacity);
/* LZ4_decompress_fast does not know the input size (lz4.c:1788); a device copy needs one.
 * `srcAvail` is the number of readable bytes at src (the Java wrapper knows it:
 * src.length - srcOff).  There is deliberately no entry point without it: the host would have to
 * read compressBound(originalSize) bytes from src, past the end of most callers' buffers.
 * One-block calls copy back exactly the bytes they produced: dst[result, dstCapacity) is not touched. */
int b200lz4_decompress_fast_bounded(const char* src, int srcAvail, char* dst, int originalSize);

uint32_t b200xxh32(const void* input, size_t len, uint32_t seed);
uint64_t b200xxh64(const void* input, size_t len, uint64_t seed);

/* streaming hash state: opaque handle (jlong on the Java side) */
void*    b200xxh32_create(uint32_t seed);
void     b200xxh32_reset(void* state, uint32_t seed);
int      b200xxh32_update(void* state, const void* input, size_t len);
uint32_t b200xxh32_digest(void* state);
void     b200xxh32_free(void* state);
void*    b200xxh64_create(uint64_t seed);
void     b200xxh64_reset(void* state, uint64_t seed);
int      b200xxh64_update(void* state, const void* input, size_t len);
uint64_t b200xxh64_digest(void* state);
void     b200xxh64_free(void* state);

/* ---------------------------------------------------------------- batches, DEVICE-resident
 * Every pointer is a device pointer on the current device; `stream` is a cudaStream_t
 * (NULL = default stream).  Block i reads  src_base + src_off[i]  (src_len[i] bytes) and
 * writes dst_base + dst_off[i] (at most dst_cap[i] bytes); result[i] follows the
 * single-block return convention.  The calls are asynchronous on `stream` and return 0 or
 * a B200LZ4_E_* code for launch failures.
 *
 * compress_fast: `max_src_len` is an upper bound on src_len[] chosen by the caller
 * (<= 65536 selects the 16-bit position table like lz4.c:1353; 0 = unknown -> 32-bit). */
int b200lz4_compress_fast_batch_dev(const uint8_t* src_base, const uint64_t* src_off, const int32_t* src_len,
                                    uint8_t* dst_base, const uint64_t* dst_off, const int32_t* dst_cap,
                                    int32_t* result, size_t n, int max_src_len, void* stream);
int b200lz4_compress_hc_batch_dev(const uint8_t* src_base, const uint64_t* src_off, const int32_t* src_len,
                                  uint8_t* dst_base, const uint64_t* dst_off, const int32_t* dst_cap,
                                  int32_t* result, size_t n, int level, void* stream);
int b200lz4_decompress_safe_batch_dev(const uint8_t* src_base, const uint64_t* src_off, const int32_t* src_len,
                                      uint8_t* dst_base, const uint64_t* dst_off, const int32_t* dst_cap,
                                      int32_t* result, size_t n, void* stream);
/* decompress_fast: src_avail[i] = readable bytes at the block's src; dst_len[i] = exact original size */
int b200lz4_decompress_fast_batch_dev(const uint8_t* src_base, const uint64_t* src_off, const int32_t* src_avail,
                                      uint8_t* dst_base, const uint64_t* dst_off, const int32_t* dst_len,
                                      int32_t* result, size_t n, void* stream);
/* hashes: len[] may be anything >= 0; one seed for the batch (the Java API passes one seed per call) */
int b200xxh32_batch_dev(const uint8_t* base, const uint64_t* off, const int32_t* len,
                        uint32_t seed, uint32_t* out, size_t n, void* stream);
int b200xxh64_batch_dev(const uint8_t* base, const uint64_t* off, const int32_t* len,
                        uint64_t seed, uint64_t* out, size_t n, void* stream);

/* Packing on the device -- what *_compact_host does before its copy back, for callers whose blocks stay in HBM: block i's
 * lens[i] bytes (<= 0 counts as none) move from slots + slot_off[i] to out + out_off[i]; out_off[] = the exclusive prefix
 * sums of lens[], *total = their sum (device pointers all; out needs sum(lens) bytes).  Asynchronous on `stream`. */
int b200lz4_compact_dev(const uint8_t* slots, const uint64_t* slot_off, const int32_t* lens, uint8_t* out, uint64_t* out_off,
                        uint64_t* total, size_t n, void* stream);
/* Device-side stitch of per-GPU packed shards into one stream (SURVEY.md 8e / (f)-4): shard g is shard_total[g] packed bytes
 * at shard_ptr[g] in the memory of device shard_dev[g] (a HOST array of device pointers; totals on the host -- 8 bytes per
 * GPU, the only thing exchanged).  Shard g lands in dst (memory of device dst_dev, dst_capacity bytes) at the sum of the totals
 * before it, reported in shard_pos[g] (host, may be NULL): one peer copy per shard, each on a stream of its source device, all
 * in flight together (NVLink between peers, otherwise staged by the driver).  A block at out_off[i] inside shard g is at
 * shard_pos[g] + out_off[i] in dst.  The shards must be complete before the call (synchronise their producers); returns when
 * every copy has landed.  Needs no worker threads and no host buffer; the caller's current device is left as it was. */
int b200lz4_stitch_shards_dev(const void* const* shard_ptr, const int* shard_dev, const uint64_t* shard_total, int nshard,
                              void* dst, int dst_dev, size_t dst_capacity, uint64_t* shard_pos);

/* ---------------------------------------------------------------- batches, HOST buffers
 * Same contracts, but every pointer is a HOST pointer.  The library chunks the batch and
 * pipelines H2D copy / kernel / D2H copy on several streams of the current device.  Blocks
 * must be laid out in ascending, non-overlapping order in both src and dst (the natural
 * layout of a block list over a DirectByteBuffer).  Synchronous: returns when all results
 * and output bytes are in host memory.  Returns 0 or a B200LZ4_E_* code. */
int b200lz4_compress_fast_batch_host(const uint8_t* src_base, const uint64_t* src_off, const int32_t* src_len,
                                     uint8_t* dst_base, const uint64_t* dst_off, const int32_t* dst_cap,
                                     int32_t* result, size_t n, int max_src_len);
int b200lz4_compress_hc_batch_host(const uint8_t* src_base, const uint64_t* src_off, const int32_t* src_len,
                                   uint8_t* dst_base, const uint64_t* dst_off, const int32_t* dst_cap,
                                   int32_t* result, size_t n, int level);
int b200lz4_decompress_safe_batch_host(const uint8_t* src_base, const uint64_t* src_off, const int32_t* src_len,
                                       uint8_t* dst_base, const uint64_t* dst_off, const int32_t* dst_cap,
                                       int32_t* result, size_t n);
int b200lz4_decompress_fast_batch_host(const uint8_t* src_base, const uint64_t* src_off, const int32_t* src_avail,
                                       uint8_t* dst_base, const uint64_t* dst_off, const int32_t* dst_len,
                                       int32_t* result, size_t n);
int b200xxh32_batch_host(const uint8_t* base, const uint64_t* off, const int32_t* len,
                         uint32_t seed, uint32_t* out, size_t n);
int b200xxh64_batch_host(const uint8_t* base, const uint64_t* off, const int32_t* len,
                         uint64_t seed, uint64_t* out, size_t n);

/* Compact-output compress for pipelines that want one contiguous stream (e.g. a frame
 * writer): blocks are compressed and written back-to-back into dst_base; out_off[i] and
 * result[i] give each block's position and size; *total = bytes written.  dst_capacity
 * must be >= sum(compressBound(src_len[i])) only in the worst case; the call fails with
 * B200LZ4_E_ARG if the compacted stream does not fit. */
int b200lz4_compress_fast_compact_host(const uint8_t* src_base, const uint64_t* src_off, const int32_t* src_len,
                                       uint8_t* dst_base, size_t dst_capacity, uint64_t* out_off,
                                       int32_t* result, size_t n, int max_src_len, uint64_t* total);

/* ---------------------------------------------------------------- host batches, range-sharded over several GPUs
 * ONE call from ONE process (a JVM) drives `ndev` GPUs: GPU devices[g] takes the contiguous block range
 * [g*n/ndev, (g+1)*n/ndev) (sizes differ by at most one block) and runs the host pipeline above on its own streams
 * from its own worker thread; blocks are independent, so there is no exchange between the GPUs and no collective
 * (SURVEY.md 8e).  `devices` = NULL means devices 0..ndev-1.  Same layout rules and results as the single-GPU calls
 * (result[] / out[] are filled for all n blocks; byte-identical output whatever ndev is).  Returns 0, or the first
 * B200LZ4_E_* any shard reported (b200lz4_last_error() then names the device). */
int b200lz4_compress_fast_batch_host_multi(const uint8_t* src_base, const uint64_t* src_off, const int32_t* src_len,
                                           uint8_t* dst_base, const uint64_t* dst_off, const int32_t* dst_cap,
                                           int32_t* result, size_t n, int max_src_len, const int* devices, int ndev);
int b200lz4_compress_hc_batch_host_multi(const uint8_t* src_base, const uint64_t* src_off, const int32_t* src_len,
                                         uint8_t* dst_base, const uint64_t* dst_off, const int32_t* dst_cap,
                                         int32_t* result, size_t n, int level, const int* devices, int ndev);
int b200lz4_decompress_safe_batch_host_multi(const uint8_t* src_base, const uint64_t* src_off, const int32_t* src_len,
                                             uint8_t* dst_base, const uint64_t* dst_off, const int32_t* dst_cap,
                                             int32_t* result, size_t n, const int* devices, int ndev);
int b200lz4_decompress_fast_batch_host_multi(const uint8_t* src_base, const uint64_t* src_off, const int32_t* src_avail,
                                             uint8_t* dst_base, const uint64_t* dst_off, const int32_t* dst_len,
                                             int32_t* result, size_t n, const int* devices, int ndev);
/* Packed output from several GPUs: shard g's compressed blocks are packed back to back (like
 * b200lz4_compress_fast_compact_host) starting at dst_base + shard_base[g], where shard_base[g] is the sum of the 16-byte
 * aligned bounds of the blocks before the shard — known before anything is compressed, so the GPUs never wait for each
 * other.  out_off[i] is absolute in dst_base; shard_total[g] = packed bytes of shard g.  The stream is contiguous within a
 * shard and has a gap between shards: a caller writes the ndev pieces one after the other (gather write).  dst_capacity
 * must hold the aligned bounds of all blocks.  shard_base / shard_total: ndev entries each (may be NULL). */
int b200lz4_compress_fast_compact_host_multi(const uint8_t* src_base, const uint64_t* src_off, const int32_t* src_len,
                                             uint8_t* dst_base, size_t dst_capacity, uint64_t* out_off,
                                             int32_t* result, size_t n, int max_src_len, const int* devices, int ndev,
                                             uint64_t* shard_base, uint64_t* shard_total);
int b200xxh32_batch_host_multi(const uint8_t* base, const uint64_t* off, const int32_t* len, uint32_t seed,
                               uint32_t* out, size_t n, const int* devices, int ndev);
int b200xxh64_batch_host_multi(const uint8_t* base, const uint64_t* off, const int32_t* len, uint64_t seed,
                               uint64_t* out, size_t n, const int* devices, int ndev);

/* ---------------------------------------------------------------- LZ4 Frame batch decoder
 * LZ4FrameInputStream semantics (src/java/net/jpountz/lz4/LZ4FrameInputStream.java:132-321) over a buffer
 * of concatenated frames: the host indexes the container, the device verifies header/block/content
 * XXH32 checksums and decodes all blocks of all frames in batched launches.
 * Error codes (negative): -1 premature end, -2 bad magic, -3 descriptor checksum, -4 block larger than the
 * frame's maximum, -5 block checksum, -6 block decode error, -7 content checksum, -8 content size,
 * -9 dst too small, -10 unsupported descriptor, -11 (decode_dev only) every check passed but a frame has a short block
 * before its last one (flush()), so its content is not one run inside d_slots: read block b at block_off[b] for
 * block_len_out[b] bytes (b200lz4f_index_block_offsets).
 * Errors come in STREAM order, as the reader would meet them: frame by frame the descriptor hash, block by block its checksum
 * and its decode, at the EndMark content checksum then content size; a container that is cut short or malformed behind at
 * least one frame header still gets an index, what precedes the bad spot is decoded and verified first, and decode_dev then
 * returns the container's own code (-1, -2, -4, -10).
 * d_slots layout: a full block takes blockMaxSize bytes; a block that cannot fill it (a stored block, or a compressed one
 * of fewer than blockMaxSize/255 bytes) takes what it can decode to, rounded up to 16 -- slot_bytes does not grow with
 * blockMaxSize for a stream of tiny blocks. */
int64_t b200lz4f_decompress_host(const uint8_t* src, size_t srcSize, uint8_t* dst, size_t dstCapacity);
void*   b200lz4f_index_create(const uint8_t* src_host, size_t srcSize, uint64_t* slot_bytes, int* err);
/* readSingleFrame = true (LZ4FrameInputStream.java:83-91,118-123): reading stops behind the first non-skippable frame, the
 * rest of src is not looked at; *src_consumed (may be NULL) = how far the reader got. */
int64_t b200lz4f_decompress_host_single(const uint8_t* src, size_t srcSize, uint8_t* dst, size_t dstCapacity, size_t* src_consumed);
void*   b200lz4f_index_create_single(const uint8_t* src_host, size_t srcSize, uint64_t* slot_bytes, size_t* src_consumed, int* err);
/* getExpectedContentSize / isExpectedContentSizeDefined (:416-445): *content_size = what the first non-skippable frame's
 * descriptor declares, -1 if it declares none (or there are only skippable frames).  Returns 0 or a code from the list above
 * (the descriptor hash is checked, on the device like every hash here). */
int     b200lz4f_expected_content_size(const uint8_t* src, size_t srcSize, int64_t* content_size);
size_t  b200lz4f_index_frames(void* index);
size_t  b200lz4f_index_blocks(void* index);
void    b200lz4f_index_block_offsets(void* index, uint64_t* block_off);   /* b200lz4f_index_blocks() entries, bytes into d_slots */
/* An index is host data, and decode_dev only reads it: several threads may decode one index at the same time, each into its
 * own d_slots.  decode_dev runs on the calling thread's device, like every entry point: the one b200lz4_set_device chose,
 * else the device current at the thread's first call into the library; d_src and d_slots are memory of that device.  Its
 * descriptors and results go through scratch the thread keeps for its next calls.  b200lz4f_index_free makes no CUDA call. */
int64_t b200lz4f_decode_dev(void* index, const uint8_t* d_src, uint8_t* d_slots, uint64_t* frame_off, uint64_t* frame_len,
                            int32_t* block_len_out, void* stream);
void    b200lz4f_index_free(void* index);
/* The index of a container in DEVICE memory: d_src holds srcSize bytes in memory of the current device.  The same index
 * b200lz4f_index_create (single == 0) or _single (single != 0) builds from the same bytes -- same *err, *slot_bytes,
 * *src_consumed, blocks, block offsets and stream-order verdict -- and the calls above take it unchanged.  The container is
 * walked on the device; only per-frame and per-block facts come to the host, no payload byte.  Ordered after the work already
 * queued on `stream`; returns when the index is built.
 * frame_hint (HOST array of nhint offsets, may be NULL): where the caller believes frames start (b200lz4f_compress_dev's
 * frame_off).  The stretches between hints are walked in parallel, one device thread each; one frame is always walked by one
 * thread, so a single frame of many small blocks is a serial chain of dependent loads whatever the hints.  Hints need not be
 * right: any hints give the index of no hints, a wrong one only costs time.  They must be ascending and below srcSize, or
 * the call returns NULL with *err = B200LZ4_E_ARG before anything is launched. */
void*   b200lz4f_index_create_dev(const uint8_t* d_src, size_t srcSize, int single, const uint64_t* frame_hint, size_t nhint,
                                  uint64_t* slot_bytes, size_t* src_consumed, int* err, void* stream);
/* b200lz4f_decompress_host / _single with d_src and d_dst in device memory of the current device (hints as above): the same
 * total or code (-1 .. -10; -9 when dstCapacity is too small), the same content packed into d_dst[0, total).  On an error
 * d_dst is not written at all, on success nothing past total.  Besides d_dst the call needs slot_bytes of device scratch
 * (see b200lz4f_index_create_dev; about the content size rounded up to whole blocks), kept by the calling thread for its next
 * calls; a caller short of memory calls b200lz4f_index_create_dev and b200lz4f_decode_dev into a buffer of its own.
 * Ordered after the work already queued on `stream`; returns when d_dst holds the content. */
int64_t b200lz4f_decompress_dev(const uint8_t* d_src, size_t srcSize, uint8_t* d_dst, size_t dstCapacity, int single,
                                const uint64_t* frame_hint, size_t nhint, size_t* src_consumed, void* stream);
/* Device-resident LZ4 Frame reader for ns independent streams, each read as its own LZ4FrameInputStream(in, readSingleFrame).
 * Stream s is src_len[s] bytes at d_src + src_off[s], decoded to d_dst + dst_off[s] with room dst_cap[s] (all offset / length
 * / result arrays HOST; the bytes device memory of the current device).  Source ranges may overlap or leave gaps and start at
 * any byte.  result[s] is what b200lz4f_decompress_host (single == 0) or b200lz4f_decompress_host_single (single != 0) returns
 * for the same bytes and dstCapacity = dst_cap[s]: the total, or -1 .. -10 in the same stream order (descriptor hash, then
 * each block's checksum and decode, then content checksum and content size, frame by frame; then the container's own error
 * behind them; then -9).  -11 does not occur: the blocks are packed.  src_consumed[s] (may be NULL): where the reader stopped,
 * what _single reports in *src_consumed; 0 when result[s] < 0.  content_len[s] (may be NULL): what the stream decodes to when
 * room is not the limit, result[s] on success; after a -9, a call with dst_cap[s] = content_len[s] does not return -9; 0 after
 * any other error.  A stream with result[s] < 0 writes nothing in d_dst; one that succeeds writes nothing outside
 * [dst_off[s], dst_off[s] + result[s]): every verdict is in before anything is packed.
 * Returns 0 or B200LZ4_E_*: NULL pointers where bytes or results are needed, ns above 2^31 - 1 or a destination range that
 * overflows are found before anything is launched; more than 2^31 - 1 blocks or frames in all (or one stream needing more
 * than 32 GiB of decode slots) after the first walk, before any payload is touched.  The number of launches does not depend
 * on ns or on the number of frames or blocks; per stream only its arguments go up and its results come back, and a few
 * totals in between: no block record crosses to the host.  Each stream is walked by one device thread, twice, so one long
 * stream of many small blocks is a serial chain of loads; for one large container b200lz4f_decompress_dev with hints is the
 * better call.  Ordered after the work already queued on `stream`; returns when the results are on the host.  Grow-or-keep
 * scratch of the thread's context: the frame reader's segment buffers, record regions and decode slots (about the content
 * size rounded up to whole blocks). */
int     b200lz4f_decompress_streams_dev(const uint8_t* d_src, const uint64_t* src_off, const uint64_t* src_len, size_t ns,
                                        uint8_t* d_dst, const uint64_t* dst_off, const uint64_t* dst_cap, int single,
                                        int64_t* result, uint64_t* src_consumed, uint64_t* content_len, void* stream);
/* Incremental device-resident LZ4 Frame reader for ns streams, each one LZ4FrameInputStream(in, readSingleFrame) whose bytes
 * arrive in pieces: the incremental counterpart of b200lz4f_decompress_streams_dev, built from the same parts.  A reader
 * (b200lz4f_reader_create, ns above 2^31 - 1: NULL with *err = B200LZ4_E_ARG) is host data, about 80 bytes of state per
 * stream; create and free make no CUDA call.  Any thread may use a reader, one at a time (it is not thread-safe, like
 * LZ4FrameInputStream).
 * b200lz4f_reader_read_dev: stream s's next piece is src_len[s] bytes at d_src + src_off[s]; its content goes to d_dst +
 * dst_off[s] with room dst_cap[s]; eof[s] != 0 says the piece ends the stream (HOST arrays of ns entries; the bytes device
 * memory of the current device).  Per stream:
 *  - The call takes the complete units at the start of the piece, in stream order, and stops in front of the first
 *    incomplete one.  A unit is a frame header (magic to HC byte), a block (word, payload and block checksum), the EndMark with
 *    its content checksum, or a skippable frame's 8-byte header; a skippable frame's payload is taken in any portions.
 *    src_consumed[s] is where it stopped: the next piece must start at that byte of the stream.  The reader keeps no payload
 *    byte between calls.
 *  - The content is packed into [dst_off[s], dst_off[s] + produced[s]).  A block is taken only while the room left holds its
 *    slot bound (a stored block its size, a compressed one min(blockMaxSize, 255 * its size)), so nothing is written outside
 *    that range and there is no -9.  With dst_cap[s] >= the frame's blockMaxSize every call with a complete unit progresses.
 *  - status[s]: B200LZ4F_MORE_INPUT (need[s] = the bytes from src_consumed the next unit takes, or those that make its length
 *    readable), B200LZ4F_MORE_ROOM (the first block the call could take does not fit; need[s] = its slot bound),
 *    B200LZ4F_DONE (the stream ended on a frame boundary with eof, or with single != 0 behind the first non-skippable frame),
 *    or -1 .. -10 as for b200lz4f_decompress_host: an incomplete unit with eof is -1, and a stream with no frame at all is
 *    what the host reader gives it.  Errors come in stream order: the blocks in front of the failing unit are delivered and
 *    counted in produced[s] (what LZ4FrameInputStream returns before it throws), the failing block writes nothing, and a -7
 *    or -8 comes after the frame's whole content; src_consumed[s] is where the failing unit starts.  DONE and every error
 *    are latched: later calls return the same status and take and produce nothing.
 *  - Whatever the pieces and room, the concatenated content and the final status are what b200lz4f_decompress_host /
 *    _single returns for the whole stream, with the same total src_consumed.  The content checksum (four lanes, an open
 *    stripe, a 64-bit length) and the content count travel in the state, so frames above 4 GiB are checked.
 * Returns 0 or B200LZ4_E_*: a NULL reader or pointer, ns other than the reader's, or a destination range that overflows are
 * found before anything is launched; more than 2^31 - 1 blocks or frames in one call after the first walk.  The number of
 * launches does not depend on ns or on the number of frames or blocks; two synchronisations (scan totals, end); only the
 * per-stream arguments, states and results and a few totals cross to and from the host, no block record and no payload
 * byte.  Ordered after the work already queued on `stream`; returns when the results are on the host.  Grow-or-keep scratch
 * of the thread's context (the frame reader's segment buffers, record regions and decode slots), sized by the call -- the
 * pieces, the blocks taken, the room -- never by how long a stream has been read. */
/* The statuses of the incremental frame calls, and of the incremental LZ4Block calls too (b200lz4block_writer_* /
 * b200lz4block_reader_*) */
#define B200LZ4F_MORE_INPUT 0
#define B200LZ4F_MORE_ROOM  1
#define B200LZ4F_DONE       2
void*   b200lz4f_reader_create(size_t ns, int single, int* err);
int     b200lz4f_reader_read_dev(void* reader, const uint8_t* d_src, const uint64_t* src_off, const uint64_t* src_len,
                                 const uint8_t* eof, uint8_t* d_dst, const uint64_t* dst_off, const uint64_t* dst_cap,
                                 int32_t* status, uint64_t* src_consumed, uint64_t* produced, uint64_t* need, void* stream);
void    b200lz4f_reader_free(void* reader);
/* Device-resident LZ4 Frame writer (LZ4FrameOutputStream.java:178-251) for nf independent frames, with bsCode / flags /
 * hc_level as b200lz4f_compress_host_hc takes them.  Frame f is src_len[f] bytes at d_src + src_off[f] (src_off / src_len:
 * HOST arrays of nf entries; the bytes are in device memory of the current device).  The frames are written back to back
 * into d_dst (device, dst_capacity bytes); frame_off[f] / frame_len[f] (host, may be NULL) say where.  b200lz4f_compress_host_hc
 * is this writer run on a device copy of its source at the source's 16-byte phase, so each frame is byte for byte the one it
 * writes for the same bytes at the same phase.  Ordered after the work already queued on `stream`; returns when the frames
 * are in d_dst.
 * Returns the total bytes written, or: -9 dst_capacity < sum of b200lz4f_compress_bound(src_len[f], bsCode);
 * -10 content checksum requested for a frame longer than 0x7FFFFFFF bytes; B200LZ4_E_ARG, _CUDA, _NODEVICE.  Argument and
 * size errors are found before anything is launched or written. */
int64_t b200lz4f_compress_dev(const uint8_t* d_src, const uint64_t* src_off, const uint64_t* src_len, size_t nf,
                              uint8_t* d_dst, size_t dst_capacity, uint64_t* frame_off, uint64_t* frame_len,
                              int bsCode, int flags, int hc_level, void* stream);
/* Incremental device-resident LZ4 Frame writer for ns streams, each one LZ4FrameOutputStream(out, BLOCKSIZE(bsCode),
 * knownSize, compressor, bits) whose content arrives in pieces (LZ4FrameOutputStream.java:178-306): the incremental
 * counterpart of b200lz4f_compress_dev, built from the same parts.  bsCode / flags / hc_level as b200lz4f_compress_dev takes
 * them, for every stream.  A writer (b200lz4f_writer_create) is host data, a few dozen bytes of state per stream; create and
 * free make no CUDA call.  It returns NULL with *err = B200LZ4_E_ARG for a bsCode outside 4..7, ns above 2^31 - 1, or, with
 * flags bit 2, a NULL known_size (HOST array of ns declared content sizes) or an entry below 0 (the constructor's
 * IllegalArgumentException).  Any thread may use a writer, one at a time (it is not thread-safe, like LZ4FrameOutputStream).
 * b200lz4f_writer_write_dev: stream s's next piece is src_len[s] bytes at d_src + src_off[s]; its frame bytes go to d_dst +
 * dst_off[s] with room dst_cap[s]; op[s] is B200LZ4F_WRITE, _FLUSH or _CLOSE (HOST arrays of ns entries; the bytes device
 * memory of the current device).  Per stream:
 *  - The stream's first call with room for it writes the header (content size known_size[s]).  Then the call takes whole
 *    blocks of blockMaxSize from the start of the piece; with FLUSH or CLOSE the rest of the piece as one short block (none
 *    when nothing is left, as flush() writes none); with CLOSE then the EndMark and the content checksum.
 *  - A unit is taken only while the room left holds its bound: a block 4 + its length (+ 4 with block checksums), the header
 *    7 or 15 bytes, the EndMark 4 or 8.  The bytes go to [dst_off[s], dst_off[s] + produced[s]), never past dst_cap[s].
 *  - src_consumed[s] is the bytes taken.  The rest of the piece is the caller's to present again at the start of the next
 *    one: the writer keeps no payload byte between calls.
 *  - status[s]: B200LZ4F_MORE_INPUT (everything takeable was taken; need[s] = the bytes missing for the next whole block,
 *    blockMaxSize after a flush), B200LZ4F_MORE_ROOM (need[s] = the bound of the unit that did not fit; a CLOSE that ran out
 *    of room is repeated), B200LZ4F_DONE (closed; latched: later calls take and produce nothing).  known_size is not checked
 *    against the content, as LZ4FrameOutputStream does not check it: a mismatch gives a frame the readers answer with -8.
 *  - The concatenated output of stream s is byte for byte what LZ4FrameOutputStream writes for the same content with
 *    flush() where FLUSH was passed, each block compressed by the library's block compressor at the 16-byte phase where the
 *    call found it; with no FLUSH and pieces at the phase of the whole content, the frame b200lz4f_compress_dev writes for it.
 *    The content checksum travels in the state, so frames of any length are checksummed.
 * Returns 0 or B200LZ4_E_*: a NULL writer or pointer, an op above _CLOSE, a destination range that overflows or more than
 * 2^31 - 1 blocks in one call are found before anything is launched or written.  The launches depend on the number of
 * chunks, not on ns or the number of blocks; one synchronisation; only the plan, the ranges written and the checksum states
 * cross PCIe.  Ordered after the work already queued on `stream`; returns when the results are on the host.  Grow-or-keep
 * scratch of the thread's context (the frame writer's), sized by the call, never by how much a stream has written. */
/* The ops of the incremental frame writer, and of the incremental LZ4Block writer too (b200lz4block_writer_*: FLUSH is
 * flush() with syncFlush = true, CLOSE is finish() and its end block) */
#define B200LZ4F_WRITE 0      /* take whole blocks only                                  */
#define B200LZ4F_FLUSH 1      /* ... and the rest of the piece as a short block (flush()) */
#define B200LZ4F_CLOSE 2      /* ... then the EndMark and content checksum (close())      */
void*   b200lz4f_writer_create(size_t ns, int bsCode, int flags, int hc_level, const int64_t* known_size, int* err);
int     b200lz4f_writer_write_dev(void* writer, const uint8_t* d_src, const uint64_t* src_off, const uint64_t* src_len,
                                  const uint8_t* op, uint8_t* d_dst, const uint64_t* dst_off, const uint64_t* dst_cap,
                                  int32_t* status, uint64_t* src_consumed, uint64_t* produced, uint64_t* need, void* stream);
void    b200lz4f_writer_free(void* writer);

/* ---------------------------------------------------------------- lz4-java's containers as whole-buffer calls
 * LZ4 Frame writer (LZ4FrameOutputStream.java:178-251): independent blocks of 64 KiB..4 MiB (bsCode 4..7), blocks that
 * do not shrink are stored raw; flags bit0 = content checksum, bit1 = block checksums, bit2 = content size.
 * "LZ4Block" container (LZ4BlockOutputStream.java:203-266 / LZ4BlockInputStream.java:191-264): 21-byte block
 * headers, XXH32 (seed 0x9747b28c, 28-bit) of each original block, fast decompressor on the read side.
 * Length-prefixed blocks (LZ4CompressorWithLength / LZ4DecompressorWithLength).
 * Return: bytes written / decoded, or negative: -1 premature end, -2 corrupted, -9 dst too small, B200LZ4_E_*. */
size_t  b200lz4f_compress_bound(size_t srcSize, int bsCode);
/* The frame is written on the calling thread's device by b200lz4f_compress_dev, from a copy of src staged at src's 16-byte
 * phase.  Besides b200lz4f_compress_dev's scratch, the call needs srcSize + b200lz4f_compress_bound(srcSize, bsCode) (plus up
 * to 30) bytes of device memory for that copy and the frame, and the thread keeps them for its next calls. */
int64_t b200lz4f_compress_host(const uint8_t* src, size_t srcSize, uint8_t* dst, size_t dstCapacity, int bsCode, int flags);
/* the writers' LZ4Compressor argument (LZ4FrameOutputStream.java:132-133, LZ4BlockOutputStream.java:96,124): hc_level 0 = the
 * fast compressor (what the calls without _hc use), 1..17 = LZ4_compress_HC at that level */
int64_t b200lz4f_compress_host_hc(const uint8_t* src, size_t srcSize, uint8_t* dst, size_t dstCapacity, int bsCode, int flags, int hc_level);
size_t  b200lz4block_compress_bound(size_t srcSize, int blockSize);
int64_t b200lz4block_compress_host(const uint8_t* src, size_t srcSize, uint8_t* dst, size_t dstCapacity, int blockSize);
int64_t b200lz4block_compress_host_hc(const uint8_t* src, size_t srcSize, uint8_t* dst, size_t dstCapacity, int blockSize, int hc_level);
/* stopOnEmptyBlock: LZ4BlockInputStream's constructor flag (LZ4BlockInputStream.java:60-72; its default is true): non-zero
 * ends at the first empty block and reports in *srcConsumed (may be NULL) how far it read; zero steps over empty blocks and
 * reads concatenated streams to the end of src. */
int64_t b200lz4block_decompress_host(const uint8_t* src, size_t srcSize, uint8_t* dst, size_t dstCapacity,
                                     int stopOnEmptyBlock, size_t* srcConsumed);

/* Device-resident LZ4Block writer (LZ4BlockOutputStream.java:203-266) for ns independent streams.  Stream s is src_len[s]
 * bytes at d_src + src_off[s] (HOST arrays; the bytes are in device memory of the current device); the streams are written
 * back to back into d_dst, stream_off / stream_len (host, may be NULL) say where.  Each stream is byte for byte what
 * b200lz4block_compress_host_hc writes for the same bytes at the same 16-byte phase (that call is this writer run on a device
 * copy of its source).  blockSize 64..32 MiB (any value; the token's level nibble comes from it), hc_level 0 = the fast
 * compressor, 1..17 = LZ4_compress_HC at that level.  Returns the total bytes written, or: -9 dst_capacity < sum of
 * b200lz4block_compress_bound(src_len[s], blockSize); B200LZ4_E_ARG, _CUDA, _NODEVICE.  Argument and size errors are found
 * before anything is launched or written.  Ordered after the work already queued on `stream`; returns when the streams are
 * in d_dst.  Grow-or-keep scratch of the thread's context: the frame writer's. */
int64_t b200lz4block_compress_dev(const uint8_t* d_src, const uint64_t* src_off, const uint64_t* src_len, size_t ns,
                                  uint8_t* d_dst, size_t dst_capacity, uint64_t* stream_off, uint64_t* stream_len,
                                  int blockSize, int hc_level, void* stream);

/* Device-resident LZ4Block reader (LZ4BlockInputStream.java:191-264) for ns independent streams, each read as its own
 * LZ4BlockInputStream(in, stopOnEmptyBlock).  Stream s: src_len[s] bytes at d_src + src_off[s], decoded to d_dst + dst_off[s]
 * with room dst_cap[s] (all offset / length arrays HOST, the bytes device memory of the current device).  result[s] is what
 * b200lz4block_decompress_host returns for the same bytes and capacity, src_consumed[s] (may be NULL) what it reports in
 * *srcConsumed (0 when result[s] < 0).  content_len[s] (may be NULL): what the stream decodes to when room is not the limit;
 * it equals result[s] when result[s] >= 0, and when result[s] == -9 a second call with dst_cap[s] = content_len[s] does not
 * return -9.  On success nothing in d_dst outside [dst_off[s], dst_off[s] + result[s]) is written for stream s; on an error
 * [dst_off[s], dst_off[s] + dst_cap[s]) holds unspecified bytes and nothing outside it is written.  No payload byte crosses to
 * the host: per stream its arguments go up and its results come back, and two block counts in between.  Returns 0 or
 * B200LZ4_E_*: NULL pointers where bytes or results are needed, ns above 2^31 - 1 or a destination range that overflows are
 * found before anything is launched.  Ordered after the work already queued on `stream`; returns when the results are on the
 * host.  Grow-or-keep scratch of the thread's context: the frame reader's. */
int     b200lz4block_decompress_dev(const uint8_t* d_src, const uint64_t* src_off, const uint64_t* src_len, size_t ns,
                                    uint8_t* d_dst, const uint64_t* dst_off, const uint64_t* dst_cap, int stopOnEmptyBlock,
                                    int64_t* result, uint64_t* src_consumed, uint64_t* content_len, void* stream);
/* Incremental device-resident LZ4Block writer for ns streams, each one LZ4BlockOutputStream(out, blockSize, compressor,
 * XXHash32 seed 0x9747b28c, syncFlush) whose content arrives in pieces (LZ4BlockOutputStream.java:160-266): the incremental
 * counterpart of b200lz4block_compress_dev, built from the same parts.  blockSize / hc_level as b200lz4block_compress_dev
 * takes them, for every stream.  The ops and statuses are the frame calls': B200LZ4F_WRITE / _FLUSH / _CLOSE and
 * B200LZ4F_MORE_INPUT / _MORE_ROOM / _DONE.  A writer (b200lz4block_writer_create) is host data, one byte of state per
 * stream (whether it is closed); create and free make no CUDA call.  It returns NULL with *err = B200LZ4_E_ARG for a
 * blockSize outside 64..32 MiB or ns above 2^31 - 1.  Any thread may use a writer, one at a time (it is not thread-safe,
 * like LZ4BlockOutputStream).
 * b200lz4block_writer_write_dev: stream s's next piece is src_len[s] bytes at d_src + src_off[s]; its stream bytes go to
 * d_dst + dst_off[s] with room dst_cap[s]; op[s] is B200LZ4F_WRITE, _FLUSH or _CLOSE (HOST arrays of ns entries; the bytes
 * device memory of the current device).  Per stream:
 *  - The call takes whole blocks of blockSize from the start of the piece; with FLUSH (flush() with syncFlush = true) or
 *    CLOSE (finish()) the rest of the piece as one short block (none when nothing is left); with CLOSE then the 21-byte
 *    empty end block.
 *  - A unit is taken only while the room left holds its bound: a block 21 + its length (a block that does not shrink is
 *    stored), the end block 21.  The bytes go to [dst_off[s], dst_off[s] + produced[s]), never past dst_cap[s].
 *  - src_consumed[s] is the bytes taken.  The rest of the piece is the caller's to present again at the start of the next
 *    one: the writer keeps no payload byte between calls.
 *  - status[s]: B200LZ4F_MORE_INPUT (need[s] = the bytes missing for the next whole block, blockSize after a flush),
 *    B200LZ4F_MORE_ROOM (need[s] = the bound of the unit that did not fit), B200LZ4F_DONE (closed; latched: later calls
 *    take and produce nothing).
 *  - The concatenated output of stream s is byte for byte what LZ4BlockOutputStream writes for the same content with
 *    syncFlush and flush() where FLUSH was passed, each block compressed by the library's block compressor at the 16-byte
 *    phase where the call found it; with no FLUSH and pieces at the phase of the whole content, the stream
 *    b200lz4block_compress_dev writes for it.
 * Returns 0 or B200LZ4_E_*: a NULL writer or pointer, an op above _CLOSE, a destination range that overflows or more than
 * 2^31 - 1 blocks in one call are found before anything is launched or written.  The launches depend on the number of
 * chunks, not on ns or the number of blocks; one synchronisation; only the plan and the ranges written cross PCIe.  Ordered
 * after the work already queued on `stream`; returns when the results are on the host.  Grow-or-keep scratch of the
 * thread's context (the frame writer's), sized by the call, never by how much a stream has written. */
void*   b200lz4block_writer_create(size_t ns, int blockSize, int hc_level, int* err);
int     b200lz4block_writer_write_dev(void* writer, const uint8_t* d_src, const uint64_t* src_off, const uint64_t* src_len,
                                      const uint8_t* op, uint8_t* d_dst, const uint64_t* dst_off, const uint64_t* dst_cap,
                                      int32_t* status, uint64_t* src_consumed, uint64_t* produced, uint64_t* need, void* stream);
void    b200lz4block_writer_free(void* writer);
/* Incremental device-resident LZ4Block reader for ns streams, each one LZ4BlockInputStream(in, stopOnEmptyBlock) whose bytes
 * arrive in pieces (LZ4BlockInputStream.java:191-264): the incremental counterpart of b200lz4block_decompress_dev, built from
 * the same parts.  Statuses as for the frame calls (B200LZ4F_MORE_INPUT / _MORE_ROOM / _DONE).  A reader
 * (b200lz4block_reader_create, ns above 2^31 - 1: NULL with *err = B200LZ4_E_ARG) is host data, the latched status of each
 * stream; create and free make no CUDA call.  Any thread may use a reader, one at a time (it is not thread-safe, like
 * LZ4BlockInputStream).
 * b200lz4block_reader_read_dev: stream s's next piece is src_len[s] bytes at d_src + src_off[s]; its content goes to d_dst +
 * dst_off[s] with room dst_cap[s]; eof[s] != 0 says the piece ends the stream (HOST arrays of ns entries; the bytes device
 * memory of the current device).  Per stream:
 *  - The call takes the complete units (a 21-byte block header with its payload) at the start of the piece, in stream
 *    order, and decodes them straight into [dst_off[s], dst_off[s] + produced[s]).  It stops in front of the first unit the
 *    piece holds only in part, and in front of the first block whose original length is above the room left: room is exact,
 *    so there is no -9, and with dst_cap[s] >= the largest block every call with a complete unit progresses.
 *    src_consumed[s] is where it stopped: the next piece must start at that byte of the stream.
 *  - status[s]: B200LZ4F_MORE_INPUT (need[s] = the unit's length once its header is readable, else 21), B200LZ4F_MORE_ROOM
 *    (need[s] = the block's original length), B200LZ4F_DONE (the first empty block with stopOnEmptyBlock; without it, eof
 *    on a block boundary or inside a header, as LZ4BlockInputStream's tryReadFully ends quietly), or -1 / -2 as
 *    b200lz4block_decompress_host returns them: an incomplete payload with eof is -1.  Errors come in stream order: the
 *    blocks in front of the failing unit (a bad header, a failed decode or a wrong checksum) are delivered and counted in
 *    produced[s], and src_consumed[s] is where the failing unit starts.  DONE and every error are latched: later calls
 *    return the same status and take and produce nothing.
 *  - After an error [dst_off[s] + produced[s], dst_off[s] + dst_cap[s]) holds unspecified bytes; nothing outside the
 *    stream's range is ever written, and a call without an error writes nothing past produced[s].
 *  - Whatever the pieces and room, the concatenated content, the final status and the total src_consumed are what
 *    b200lz4block_decompress_host gives for the whole stream with ample room.
 * Returns 0 or B200LZ4_E_*: a NULL reader or pointer, or a destination range that overflows are found before anything is
 * launched.  The number of launches does not depend on ns or on the number of blocks; two synchronisations (scan totals,
 * end); only the per-stream arguments, states and results and two totals cross to and from the host.  Ordered after the
 * work already queued on `stream`; returns when the results are on the host.  Grow-or-keep scratch of the thread's context
 * (the frame reader's segment buffers and record regions), sized by the call, never by how long a stream has been read. */
void*   b200lz4block_reader_create(size_t ns, int stopOnEmptyBlock, int* err);
int     b200lz4block_reader_read_dev(void* reader, const uint8_t* d_src, const uint64_t* src_off, const uint64_t* src_len,
                                     const uint8_t* eof, uint8_t* d_dst, const uint64_t* dst_off, const uint64_t* dst_cap,
                                     int32_t* status, uint64_t* src_consumed, uint64_t* produced, uint64_t* need, void* stream);
void    b200lz4block_reader_free(void* reader);
int     b200lz4_compress_with_length(const char* src, char* dst, int srcSize, int dstCapacity);
int     b200lz4_decompressed_length(const char* src);
int     b200lz4_decompress_with_length(const char* src, int srcAvail, char* dst, int dstCapacity);
/* LZ4DecompressorWithLength(LZ4SafeDecompressor) (lz4-java 1.8, LZ4DecompressorWithLength.java:148-154): src is exactly one
 * record of srcLen bytes.  -1 when srcLen < 4, or the declared length is negative or larger than dstCapacity; otherwise
 * b200lz4_decompress_safe(src + 4, dst, srcLen - 4, declared): the bytes decoded, or < 0. */
int     b200lz4_decompress_with_length_safe(const char* src, int srcLen, char* dst, int dstCapacity);

/* Device-resident LZ4CompressorWithLength (LZ4CompressorWithLength.java:45-50) for n independent records.  Record r is
 * src_len[r] bytes at d_src + src_off[r] (HOST arrays; the bytes are in device memory of the current device); the records are
 * written back to back into d_dst, rec_off / rec_len (host, may be NULL) say where.  A record is 4 bytes of little-endian
 * src_len[r], then one LZ4 block of the whole record.  hc_level 0 = the fast compressor: each record is byte for byte what
 * b200lz4_compress_with_length writes for the same bytes at the same 16-byte phase (the compressor is picked per record by its
 * length, as that call picks it).  1..17 = LZ4_compress_HC at that level: the block is what b200lz4_compress_HC writes.
 * Returns the total bytes written, or: -9 dst_capacity < sum of b200lz4_compressBound(src_len[r]) + 4; B200LZ4_E_ARG
 * (a record longer than 0x7E000000 bytes, a NULL pointer where bytes are needed), _CUDA, _NODEVICE.  Argument and size errors
 * are found before anything is launched or written.  Ordered after the work already queued on `stream`; returns when the
 * records are in d_dst.  Grow-or-keep scratch of the thread's context: the frame writer's. */
int64_t b200lz4_compress_with_length_dev(const uint8_t* d_src, const uint64_t* src_off, const uint64_t* src_len, size_t n,
                                         uint8_t* d_dst, size_t dst_capacity, uint64_t* rec_off, uint64_t* rec_len,
                                         int hc_level, void* stream);

/* Device-resident LZ4DecompressorWithLength for n independent records, HBM to HBM.  Record r is the src_len[r] readable bytes
 * at d_src + src_off[r] (at most 2^31 - 1), decoded to d_dst + dst_off[r] with room dst_cap[r] (all offset / length arrays HOST,
 * the bytes device memory of the current device).  safe == 0, the LZ4FastDecompressor flavour: result[r] is what
 * b200lz4_decompress_with_length(src, src_len, dst, dst_cap) returns (the bytes read including the prefix, or < 0);
 * safe != 0, the LZ4SafeDecompressor flavour: what b200lz4_decompress_with_length_safe returns (the bytes decoded, or < 0).
 * orig_len[r] (may be NULL): the declared length, -1 when src_len[r] < 4; a record refused for want of room can be read again
 * with dst_cap[r] = orig_len[r].  Nothing outside [dst_off[r], dst_off[r] + dst_cap[r]) is written, nothing at all for a
 * record its header rejects, and on success nothing past dst_off[r] + the declared length (fast) or + result[r] (safe).
 * Three launches whatever n is; only the per-record arguments go up and the results come back.  Returns 0 or B200LZ4_E_*:
 * NULL pointers where bytes or results are needed, n above 2^31 - 1, a record above 2^31 - 1 bytes or a destination range
 * that overflows are found before anything is launched.  Ordered after the work already queued on `stream`; returns when
 * the results are on the host.  Grow-or-keep scratch of the thread's context: the frame reader's. */
int     b200lz4_decompress_with_length_dev(const uint8_t* d_src, const uint64_t* src_off, const uint64_t* src_len, size_t n,
                                           uint8_t* d_dst, const uint64_t* dst_off, const uint64_t* dst_cap, int safe,
                                           int64_t* result, int64_t* orig_len, void* stream);

/* kernel-launch counter (bench.py's "gpu_launches"): number of kernels this library has
 * launched from the calling process since load / since the last reset. */
uint64_t b200lz4_launch_count(void);
void     b200lz4_launch_count_reset(void);

/* pipeline contexts (3 streams + device staging each) created in this process so far.  A thread keeps one per device;
 * contexts of threads that exited are reused by new threads, so with the reference's usage (any number of Java threads
 * calling the singleton codecs, LZ4Compressor.java:25) this stays at the peak number of CONCURRENT callers. */
int      b200lz4_context_count(void);

#ifdef __cplusplus
}
#endif
#endif /* B200LZ4_H */
