/*
 * zstdb200.h -- C ABI of the GPU-native (H100) Zstandard block codec (libzstdb200.so).
 *
 * Two layers are exported, both plain C (pointers + sizes, no torch / C++ types):
 *
 *  (1) the libzstd entry points that luben/zstd-jni's JNI glue binds for the hot path
 *      (SURVEY.md section 8b).  Signatures, ownership and the error convention are those of
 *      the reference's src/main/native/zstd.h, so the unmodified jni_*.c link against this
 *      library instead of the bundled libzstd.  Each declaration cites the JNI call site it
 *      serves (N/ = luben/zstd-jni src/main/native/).
 *
 *  (2) a batch API (zstdb200_*) that the same glue -- or any other host -- uses to hand
 *      the GPU what it is good at: thousands of independent <=128 KB chunks per call.
 *      Every chunk becomes one frame, byte-identical to ZSTD_compress2(chunk, level).
 *
 * Error convention (N/common/error_private.h:49-54): functions return size_t; a value
 * greater than (size_t)-ZSTD_error_maxCode is -(error code), see ZSTD_isError().
 * There is NO CPU fallback: if no CUDA device is usable the calls fail with
 * ZSTD_error_GENERIC (code 1) and zstdb200_last_error() says why.
 */
#ifndef ZSTDB200_H
#define ZSTDB200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ZSTDB200_API __attribute__((visibility("default")))

/* ------------------------------------------------------------------------------------
 * (1) libzstd-compatible entry points
 * ---------------------------------------------------------------------------------- */
typedef struct ZSTD_CCtx_s ZSTD_CCtx;
typedef struct ZSTD_DCtx_s ZSTD_DCtx;
typedef ZSTD_CCtx ZSTD_CStream;
typedef ZSTD_DCtx ZSTD_DStream;

/* values of N/zstd.h:492-545 (ZSTD_cParameter) that the JNI glue sets on this path */
typedef enum {
    ZSTD_c_compressionLevel = 100,
    ZSTD_c_windowLog = 101, ZSTD_c_hashLog = 102, ZSTD_c_chainLog = 103, ZSTD_c_searchLog = 104,
    ZSTD_c_minMatch = 105, ZSTD_c_targetLength = 106, ZSTD_c_strategy = 107,
    ZSTD_c_contentSizeFlag = 200,
    ZSTD_c_checksumFlag = 201,
    ZSTD_c_dictIDFlag = 202,
    ZSTD_c_nbWorkers = 400,
    ZSTD_c_format = 10,                 /* ZSTD_c_experimentalParam2 (N/zstd.h:2051): ZSTD_f_zstd1 / ZSTD_f_zstd1_magicless, N/jni_zstd.c:362-363 */
    /* extension of this library (not in libzstd): when non-zero, ZSTD_compress2 / ZSTD_compressCCtx accept inputs larger
     * than one block and write them as one independent frame per 128 KB -- a legal zstd stream (every decoder reads
     * concatenated frames) but NOT the bytes the reference would produce.  Off by default: without it such inputs are
     * refused with ZSTD_error_parameter_unsupported.  Environment default: ZSTDB200_MULTIFRAME=1. */
    ZSTDB200_c_multiFrame = 0xB200
} ZSTD_cParameter;
/* N/zstd.h:642-672 (ZSTD_dParameter): the two the JNI glue sets on this path, N/jni_zstd.c:403,413-414 */
typedef enum { ZSTD_d_windowLogMax = 100, ZSTD_d_format = 1000 /* ZSTD_d_experimentalParam1 */ } ZSTD_dParameter;
typedef enum { ZSTD_f_zstd1 = 0, ZSTD_f_zstd1_magicless = 1 } ZSTD_format_e;        /* N/zstd.h:1382-1389 */
typedef enum { ZSTD_reset_session_only = 1, ZSTD_reset_parameters = 2, ZSTD_reset_session_and_parameters = 3 } ZSTD_ResetDirective;
typedef enum { ZSTD_e_continue = 0, ZSTD_e_flush = 1, ZSTD_e_end = 2 } ZSTD_EndDirective;
typedef struct { const void* src; size_t size; size_t pos; } ZSTD_inBuffer;    /* N/zstd.h:731-735 */
typedef struct { void* dst; size_t size; size_t pos; } ZSTD_outBuffer;         /* N/zstd.h:737-741 */

#define ZSTD_CONTENTSIZE_UNKNOWN (0ULL - 1)
#define ZSTD_CONTENTSIZE_ERROR (0ULL - 2)

/* N/jni_zstd.c:573-667 (error-code getters), N/jni_fast_zstd.c (every call site checks ZSTD_isError) */
ZSTDB200_API unsigned ZSTD_isError(size_t code);
ZSTDB200_API const char* ZSTD_getErrorName(size_t code);
ZSTDB200_API int ZSTD_getErrorCode(size_t code);          /* returns the positive ZSTD_ErrorCode */
ZSTDB200_API unsigned ZSTD_versionNumber(void);           /* 10507 */
ZSTDB200_API const char* ZSTD_versionString(void);        /* "1.5.7" */
ZSTDB200_API int ZSTD_minCLevel(void);                    /* N/jni_zstd.c: minCompressionLevel */
ZSTDB200_API int ZSTD_maxCLevel(void);
ZSTDB200_API int ZSTD_defaultCLevel(void);

/* N/jni_zstd.c:compressBound -> ZSTD_compressBound (N/zstd.h:249) */
ZSTDB200_API size_t ZSTD_compressBound(size_t srcSize);

/* contexts: N/jni_fast_zstd.c:253-258 (init -> ZSTD_createCCtx), :268-275 (free), :683-696 (DCtx) */
ZSTDB200_API ZSTD_CCtx* ZSTD_createCCtx(void);
ZSTDB200_API size_t ZSTD_freeCCtx(ZSTD_CCtx* cctx);
ZSTDB200_API ZSTD_DCtx* ZSTD_createDCtx(void);
ZSTDB200_API size_t ZSTD_freeDCtx(ZSTD_DCtx* dctx);
/* N/jni_fast_zstd.c:277-318 (setLevel0/setChecksum0/setContentSize0/setDictID0), N/jni_zstd.c:349-566 */
ZSTDB200_API size_t ZSTD_CCtx_setParameter(ZSTD_CCtx* cctx, ZSTD_cParameter param, int value);
ZSTDB200_API size_t ZSTD_CCtx_reset(ZSTD_CCtx* cctx, ZSTD_ResetDirective reset);   /* N/jni_fast_zstd.c:605,633 */
ZSTDB200_API size_t ZSTD_DCtx_reset(ZSTD_DCtx* dctx, ZSTD_ResetDirective reset);   /* N/jni_fast_zstd.c:797,824 */
ZSTDB200_API size_t ZSTD_CCtx_setPledgedSrcSize(ZSTD_CCtx* cctx, unsigned long long pledgedSrcSize);
ZSTDB200_API size_t ZSTD_DCtx_setParameter(ZSTD_DCtx* dctx, ZSTD_dParameter param, int value);   /* N/jni_zstd.c:403,413-414 */
/* N/jni_fast_zstd.c:373 (J/ZstdCompressCtx.getFrameProgression); the MT fields stay 0 */
typedef struct { unsigned long long ingested, consumed, produced, flushed; unsigned currentJobID, nbActiveWorkers; } ZSTD_frameProgression;
ZSTDB200_API ZSTD_frameProgression ZSTD_getFrameProgression(const ZSTD_CCtx* cctx);

/* one-shot hot path:
 *   ZSTD_compress2       <- N/jni_fast_zstd.c:607,635 (compressDirectByteBuffer0 / compressByteArray0), N/jni_zstd.c:23
 *   ZSTD_compress        <- convenience (same frame as compress2 with a fresh ctx at `level`)
 *   ZSTD_decompressDCtx  <- N/jni_fast_zstd.c:799,826,861,895
 *   ZSTD_decompress      <- N/jni_zstd.c:62
 * src/dst are caller-owned host memory borrowed for the duration of the call.
 * Compression scope of this build: srcSize <= 128 KB per call (one block => one frame), levels whose
 * parameters select the fast / dfast parsers, greedy / lazy / lazy2 (row-based match finder for inputs > 16 KB,
 * hash chain below) or btlazy2 (binary tree): the negative levels and levels 1..12 for srcSize > 16 KB, 1..10 for
 * srcSize <= 16 KB; and the optimal parser (btopt / btultra / btultra2, levels 13..22 or ZSTD_c_strategy 7..9) for
 * srcSize <= 64 KB.  Three cases return ZSTD_error_parameter_unsupported rather than different bytes: levels 11 and 12
 * on srcSize <= 16 KB (btopt rows), the optimal parser on srcSize > 64 KB (the reference splits such blocks after
 * the parse), and optimal levels in zstdb200_generate_sequences / zstdb200_sequenceProducer.  The batch calls, the
 * begin/end pair, zstdb200_compress_device and the streams apply the rule per frame: at level 19 a stream fails on its
 * first full 128 KB block, one shorter than 64 KB succeeds.
 * Decompression accepts any zstd stream without dictionary (multi-block, multi-frame, skippable, checksum). */
ZSTDB200_API size_t ZSTD_compress2(ZSTD_CCtx* cctx, void* dst, size_t dstCapacity, const void* src, size_t srcSize);
ZSTDB200_API size_t ZSTD_compress(void* dst, size_t dstCapacity, const void* src, size_t srcSize, int compressionLevel);
ZSTDB200_API size_t ZSTD_compressCCtx(ZSTD_CCtx* cctx, void* dst, size_t dstCapacity, const void* src, size_t srcSize, int compressionLevel);
ZSTDB200_API size_t ZSTD_decompressDCtx(ZSTD_DCtx* dctx, void* dst, size_t dstCapacity, const void* src, size_t srcSize);
ZSTDB200_API size_t ZSTD_decompress(void* dst, size_t dstCapacity, const void* src, size_t compressedSize);

/* frame inspection (host-side header walks): N/jni_zstd.c:70-117 (decompressedSize / findFrameCompressedSize) */
ZSTDB200_API unsigned long long ZSTD_getFrameContentSize(const void* src, size_t srcSize);
/* frame header inspection, host side (N/zstd.h:1510-1545; N/jni_zstd.c:35 magicless sizes, :139,156 dictID of a frame) */
typedef enum { ZSTD_frame, ZSTD_skippableFrame } ZSTD_FrameType_e;
typedef struct {
    unsigned long long frameContentSize;   /* ZSTD_CONTENTSIZE_UNKNOWN when absent; size of the skippable content for a skippable frame */
    unsigned long long windowSize;
    unsigned blockSizeMax;
    ZSTD_FrameType_e frameType;
    unsigned headerSize;
    unsigned dictID;                       /* skippable frame: magic variant 0..15 */
    unsigned checksumFlag;
    unsigned _reserved1;
    unsigned _reserved2;
} ZSTD_FrameHeader;
#define ZSTD_frameHeader ZSTD_FrameHeader  /* old name, used by N/jni_zstd.c:34 */
ZSTDB200_API size_t ZSTD_getFrameHeader(ZSTD_FrameHeader* zfhPtr, const void* src, size_t srcSize);
ZSTDB200_API size_t ZSTD_getFrameHeader_advanced(ZSTD_FrameHeader* zfhPtr, const void* src, size_t srcSize, ZSTD_format_e format);
ZSTDB200_API size_t ZSTD_frameHeaderSize(const void* src, size_t srcSize);
ZSTDB200_API unsigned ZSTD_isFrame(const void* buffer, size_t size);
ZSTDB200_API unsigned ZSTD_isSkippableFrame(const void* buffer, size_t size);
ZSTDB200_API unsigned ZSTD_getDictID_fromFrame(const void* src, size_t srcSize);     /* always the frame's field; dictionaries themselves are out of scope */
ZSTDB200_API size_t ZSTD_findFrameCompressedSize(const void* src, size_t srcSize);
ZSTDB200_API unsigned long long ZSTD_decompressBound(const void* src, size_t srcSize);

/* streaming (N/jni_outputstream_zstd.c:59-123, N/jni_inputstream_zstd.c:70-93, N/jni_fast_zstd.c:406-579).
 * GPU semantics, documented in INTEGRATION.md: the compressor buffers up to one block and emits
 * every block as an independent frame ("independent-frames mode": any zstd decoder reads it, but the
 * bytes differ from the reference's single-frame stream); the decompressor buffers whole frames. */
ZSTDB200_API ZSTD_CStream* ZSTD_createCStream(void);
ZSTDB200_API size_t ZSTD_freeCStream(ZSTD_CStream* zcs);
ZSTDB200_API size_t ZSTD_initCStream(ZSTD_CStream* zcs, int compressionLevel);
ZSTDB200_API size_t ZSTD_compressStream2(ZSTD_CCtx* cctx, ZSTD_outBuffer* output, ZSTD_inBuffer* input, ZSTD_EndDirective endOp);
ZSTDB200_API size_t ZSTD_compressStream(ZSTD_CStream* zcs, ZSTD_outBuffer* output, ZSTD_inBuffer* input);
ZSTDB200_API size_t ZSTD_flushStream(ZSTD_CStream* zcs, ZSTD_outBuffer* output);
ZSTDB200_API size_t ZSTD_endStream(ZSTD_CStream* zcs, ZSTD_outBuffer* output);
ZSTDB200_API size_t ZSTD_CStreamInSize(void);
ZSTDB200_API size_t ZSTD_CStreamOutSize(void);
ZSTDB200_API ZSTD_DStream* ZSTD_createDStream(void);
ZSTDB200_API size_t ZSTD_freeDStream(ZSTD_DStream* zds);
ZSTDB200_API size_t ZSTD_initDStream(ZSTD_DStream* zds);
ZSTDB200_API size_t ZSTD_decompressStream(ZSTD_DStream* zds, ZSTD_outBuffer* output, ZSTD_inBuffer* input);
ZSTDB200_API size_t ZSTD_DStreamInSize(void);
ZSTDB200_API size_t ZSTD_DStreamOutSize(void);

/* ------------------------------------------------------------------------------------
 * (2) batch API
 * ---------------------------------------------------------------------------------- */
typedef struct zstdb200_ctx_s zstdb200_ctx;

/* A context owns one CUDA device's workspaces and a stream; it is not thread-safe (one per thread,
 * like a ZSTD_CCtx, J/ZstdCompressCtx.java:31-34).  device < 0 selects the current device. */
ZSTDB200_API zstdb200_ctx* zstdb200_create(int device);
ZSTDB200_API void zstdb200_free(zstdb200_ctx* ctx);
ZSTDB200_API const char* zstdb200_last_error(void);          /* thread-local text of the last CUDA/runtime failure */
ZSTDB200_API int zstdb200_device_count(void);
/* tuning knobs; returns 0, or -1 for an unknown name or a value out of the option's range:
 *   "enc_warps_per_sm", "dec_warps_per_sm" (any value; <= 0: as many as shared memory allows),
 *   "parse_lanes" (4|8|16|32), "parse_blocks_per_sm" (1..16), "lazy_blocks_per_sm" / "opt_blocks_per_sm" (4|6|8: residency of the
 *   levels >= 5 / optimal-parser parse kernels), "parse_est_bytes" (256..65536: prefix parsed for the cost estimate that orders the parse),
 *   "dec_pipeline" (0|1), "l2_fetch_granularity" (32|64|128),
 *   "host_slices" / "host_slices_dec" (1..64: slices of the synchronous host-memory calls; defaults 1 / 2), "timing" (0|1),
 *   "entropy_overlap" (0|1, default 1: the entropy stage is launched as a programmatic dependent of the parse and
 *   takes frames in the order their parse finishes, filling the SMs the parse's tail leaves idle),
 *   "kernel_fifo" (0|1, default 1: the kernel sections of host-memory operations queued on different work sets run
 *   one after the other in submission order -- copies still overlap them; two batches in the kernels at once only slow each other down),
 *   "seek_table" (0|1, default 0: compress_items_device writes the seekable format's seek table after every item, and
 *   decompress_ranges_device locates ranges through such tables; see those calls; no environment variable).
 * zstdb200_create reads these ten from the environment (a value the option rejects is ignored): ZSTDB200_ENC_WARPS_PER_SM,
 * ZSTDB200_DEC_WARPS_PER_SM, ZSTDB200_PARSE_LANES, ZSTDB200_PARSE_BLOCKS_PER_SM, ZSTDB200_LAZY_BLOCKS_PER_SM, ZSTDB200_PARSE_EST_BYTES,
 * ZSTDB200_L2_FETCH (l2_fetch_granularity), ZSTDB200_HOST_SLICES, ZSTDB200_ENTROPY_OVERLAP and ZSTDB200_KERNEL_FIFO. */
ZSTDB200_API int zstdb200_set_option(zstdb200_ctx* ctx, const char* name, long long value);
ZSTDB200_API unsigned long long zstdb200_kernel_launches(const zstdb200_ctx* ctx);   /* kernels launched so far */
/* frames of many blocks that the host-memory decompression calls (zstdb200_decompress_batch, zstdb200_decompress_frames and
 * zstdb200_decompress_frames_begin/_end) gave to the segment decoder: regenerated there (deferred = 0), or handed to
 * the fused kernel because the segment decoder could not vouch for them (deferred = 1: corrupted, short of capacity, wrong checksum)
 * or because the item of several frames they belong to was decoded again whole (see zstdb200_split_items) */
ZSTDB200_API unsigned long long zstdb200_segment_frames(const zstdb200_ctx* ctx, int deferred);
/* items of several frames that the host-memory decompression calls decoded frame by frame (deferred = 0: each frame as its own entry, on the
 * staged, segment or fused decoder), or decoded again whole on the fused kernel because a frame did not regenerate exactly its
 * declared size or its checksum failed (deferred = 1).  An item is split when it is a whole number of frames (skippable ones included,
 * at least two), every zstd frame but the last declares its content size, those sizes fit the item's capacity, and its frames regenerate
 * at least 32 KB each on average; and only when the device workspaces of every frame (about 0.5 MB each) can be had -- otherwise the call
 * decodes every item whole, as with dec_pipeline 0.  With dec_pipeline 0 no item is split.  On a magicless context the items are
 * magicless frames (ZSTD_f_zstd1_magicless): they have no skippable frames, and are split and decoded by the same rules. */
ZSTDB200_API unsigned long long zstdb200_split_items(const zstdb200_ctx* ctx, int deferred);

/* Frame stream: one frame of many blocks decoded segment by segment as its blocks arrive, in memory that does not depend on the
 * frame's size.  The handle keeps the frame's last window on the device (a ring of a power-of-two size, at least the window plus one
 * segment's output) with the carried decoder state, and pinned host staging for at most one segment of input and one of output; each
 * call borrows the segment workspace of the context it is given.
 *   open:   parses the frame header at src (magicless: ZSTD_f_zstd1_magicless) and returns the bytes it took, or an error code:
 *           srcSize_wrong when the header is not complete, frameParameter_windowTooLarge beyond windowMax, dictionary_wrong for a
 *           frame that names a dictionary, parameter_unsupported for a skippable frame.  *fs receives the handle.
 *   decode: takes bytes from src[*srcPos, srcSize) -- block headers, blocks, the checksum -- decodes a segment whenever
 *           zstdb200_fstream_blocks(ctx) blocks or the last block are staged, and writes what it regenerated to dst[*dstPos,
 *           dstCapacity), keeping the rest staged.  Returns 0 when the frame is done and handed out (the bytes after it are not
 *           taken), 1 when it wants more input or more room, or an error code.  Bytes of earlier segments stay handed out.
 *   stats:  0 segments regenerated by the segment decoder, 1 segments decoded on the fused decoder's resume entry (doubtful
 *           segments, or every segment with dec_pipeline 0), 2 bytes of input and output the handle holds on the host. */
typedef struct zstdb200_fstream_s zstdb200_fstream;
ZSTDB200_API unsigned zstdb200_fstream_blocks(const zstdb200_ctx* ctx);      /* blocks per segment (dec_segment_blocks) */
ZSTDB200_API size_t zstdb200_fstream_open(zstdb200_ctx* ctx, const void* src, size_t srcSize, int magicless, unsigned long long windowMax,
                                          zstdb200_fstream** fs);
ZSTDB200_API size_t zstdb200_fstream_decode(zstdb200_ctx* ctx, zstdb200_fstream* fs, const void* src, size_t srcSize, size_t* srcPos,
                                            void* dst, size_t dstCapacity, size_t* dstPos);
ZSTDB200_API unsigned long long zstdb200_fstream_stats(const zstdb200_fstream* fs, int what);
ZSTDB200_API void zstdb200_fstream_free(zstdb200_fstream* fs);
/* with option "timing" = 1 every kernel launch is bracketed by CUDA events on its stream; this returns the averages
 * since the previous call as "name:ms:count;..." (synchronises).  Used by bench.py for the roofline line. */
ZSTDB200_API size_t zstdb200_kernel_times(zstdb200_ctx* ctx, char* buf, size_t cap);

/* Host-memory batch calls (H2D, kernels, D2H inside the call; synchronous).
 * compress_chunks: `src` is cut into ceil(srcSize/chunkSize) chunks (chunkSize <= 131072); chunk i becomes
 * frame i; frames are written back to back into dst (a legal multi-frame zstd stream); frameSizes[i] receives
 * each frame's size (or its error code); *dstSize the total.  dstCapacity >= sum of ZSTD_compressBound(chunk). */
ZSTDB200_API size_t zstdb200_compress_chunks(zstdb200_ctx* ctx, int level, const void* src, size_t srcSize, size_t chunkSize,
                                             void* dst, size_t dstCapacity, size_t* frameSizes, size_t* dstSize);
/* decompress_frames: `src` holds nFrames items back to back, item i being frameSizes[i] bytes (each item = one or
 * more whole frames); item i is regenerated at dst + sum(dstSizes[0..i-1]) with capacity dstSizes[i] (in: expected
 * size, e.g. from ZSTD_getFrameContentSize; out: regenerated size or error code). */
ZSTDB200_API size_t zstdb200_decompress_frames(zstdb200_ctx* ctx, const void* src, const size_t* frameSizes, size_t nFrames,
                                               void* dst, size_t dstCapacity, size_t* dstSizes);
/* Asynchronous forms of the two calls above: `_begin` queues the copy-in, the kernels and the copy-out of the sizes on work set
 * `slot` (0 .. ZSTDB200_SLOTS-1) and returns; `_end` waits for them and (compression: copies the packed frames out, then)
 * reports like the synchronous call.  Different slots overlap: with begin(0) begin(1) end(0) begin(0) end(1) ... the copy-in of
 * batch k+1 and the copy-out of batch k-1 ride on the two copy engines while batch k is in the kernels, so a stream of batches
 * costs max(kernels, copies) per batch instead of their sum.  This is what a JNI stream loop over direct buffers
 * (N/jni_outputstream_zstd.c:59-123, N/jni_directbuffercompress_zstd.c) or bench.py's end-to-end leg drives.  Buffers must stay
 * valid and untouched between begin and end; page-locked memory (cudaHostAlloc, or zstdb200_host_register on a direct
 * buffer) makes the copies truly asynchronous.  One operation per slot at a time; a context is still single-threaded.
 * The synchronous calls run on the same work sets: compress_chunks and decompress_frames on set 0, and on set 1 too when they cut
 * the batch into slices ("host_slices" / "host_slices_dec", batches of at least 512 frames); compress_batch, decompress_batch and
 * generate_sequences on set 0.  While a `_begin` is pending on a set such a call needs, the call returns ZSTD_error_stage_wrong
 * and changes nothing. */
#define ZSTDB200_SLOTS 4
ZSTDB200_API size_t zstdb200_compress_chunks_begin(zstdb200_ctx* ctx, int slot, int level, const void* src, size_t srcSize, size_t chunkSize);
ZSTDB200_API size_t zstdb200_compress_chunks_end(zstdb200_ctx* ctx, int slot, void* dst, size_t dstCapacity, size_t* frameSizes, size_t* dstSize);
ZSTDB200_API size_t zstdb200_decompress_frames_begin(zstdb200_ctx* ctx, int slot, const void* src, const size_t* frameSizes, size_t nFrames,
                                                     void* dst, size_t dstCapacity, const size_t* dstSizes);
ZSTDB200_API size_t zstdb200_decompress_frames_end(zstdb200_ctx* ctx, int slot, size_t* dstSizes);
/* page-lock / release a caller-owned host range (a DirectByteBuffer's address range) so that the copies of the calls above run
 * on the copy engines without a staging pass; returns 0 or an error code */
ZSTDB200_API size_t zstdb200_host_register(void* ptr, size_t bytes);
ZSTDB200_API size_t zstdb200_host_unregister(void* ptr);
/* scattered host buffers (what a JNI batch entry point would pass after pinning n arrays) */
ZSTDB200_API size_t zstdb200_compress_batch(zstdb200_ctx* ctx, int level, size_t n, const void* const* src, const size_t* srcSize,
                                            void* const* dst, const size_t* dstCapacity, size_t* dstSize);
ZSTDB200_API size_t zstdb200_decompress_batch(zstdb200_ctx* ctx, size_t n, const void* const* src, const size_t* srcSize,
                                              void* const* dst, const size_t* dstCapacity, size_t* dstSize);

/* ---- entry points of features that are not built, kept here because they take THIS library's contexts (see zb_libzstd.cpp): dictionaries
 * (N/jni_zstd.c:271-346, N/jni_fast_zstd.c:133-250,325-362,673-710) and foreign sequence producers (N/jni_zstd.c:337-346).  A non-empty
 * dictionary / non-NULL CDict or DDict is refused with ZSTD_error_parameter_unsupported, clearing calls succeed; after
 * ZSTD_registerSequenceProducer(cctx, state, fn != NULL) compressions of that context report parameter_unsupported until it is cleared. */
typedef struct ZSTD_CDict_s ZSTD_CDict;
typedef struct ZSTD_DDict_s ZSTD_DDict;
typedef struct { unsigned int offset; unsigned int litLength; unsigned int matchLength; unsigned int rep; } ZSTD_Sequence;     /* N/zstd.h:1315-1350 */
typedef size_t (*ZSTD_sequenceProducer_F)(void* sequenceProducerState, ZSTD_Sequence* outSeqs, size_t outSeqsCapacity, const void* src, size_t srcSize,
                                          const void* dict, size_t dictSize, int compressionLevel, size_t windowSize);       /* N/zstd.h:2930-2936 */
ZSTDB200_API size_t ZSTD_CCtx_loadDictionary(ZSTD_CCtx* cctx, const void* dict, size_t dictSize);
ZSTDB200_API size_t ZSTD_CCtx_refCDict(ZSTD_CCtx* cctx, const ZSTD_CDict* cdict);
ZSTDB200_API size_t ZSTD_DCtx_loadDictionary(ZSTD_DCtx* dctx, const void* dict, size_t dictSize);
ZSTDB200_API size_t ZSTD_DCtx_refDDict(ZSTD_DCtx* dctx, const ZSTD_DDict* ddict);
ZSTDB200_API size_t ZSTD_compress_usingCDict(ZSTD_CCtx* cctx, void* dst, size_t dstCapacity, const void* src, size_t srcSize, const ZSTD_CDict* cdict);
ZSTDB200_API size_t ZSTD_decompress_usingDDict(ZSTD_DCtx* dctx, void* dst, size_t dstCapacity, const void* src, size_t srcSize, const ZSTD_DDict* ddict);
ZSTDB200_API void ZSTD_registerSequenceProducer(ZSTD_CCtx* cctx, void* sequenceProducerState, ZSTD_sequenceProducer_F sequenceProducer);

/* ---- sequences: the GPU match finder behind the reference's sequence-level plug points (SURVEY.md section 8f.4)
 * ZSTD_Sequence is N/zstd.h:1315-1350.  zstdb200_generate_sequences is ZSTD_generateSequences
 * (N/compress/zstd_compress.c:3520-3553) for n independent blocks of <= 128 KB: block i yields the records the reference
 * writes for a one-shot input of that size at `level` -- its sequences with raw offsets and `rep`, then the block
 * delimiter {0, last literals, 0, 0}.  nbSeqs[i] = number of records or an error code (capacity too small:
 * dstSize_tooSmall; srcSize < 7: sequenceProducer_failed and an empty block: 0 records, as in the reference). */
ZSTDB200_API size_t zstdb200_generate_sequences(zstdb200_ctx* ctx, int level, size_t n, const void* const* src, const size_t* srcSize,
                                                ZSTD_Sequence* const* outSeqs, const size_t* outSeqsCapacity, size_t* nbSeqs);
/* A block-level external sequence producer of type ZSTD_sequenceProducer_F (N/zstd.h:2820-2900), to be registered with
 * ZSTD_registerSequenceProducer -- from Java: Zstd.registerSequenceProducer / ZstdCompressCtx.registerSequenceProducer
 * with a J/SequenceProducer.java whose getFunctionPointer() returns &zstdb200_sequenceProducer and whose createState() /
 * freeState() call the two functions below (N/jni_zstd.c registerSequenceProducer, N/jni_fast_zstd.c).  libzstd keeps
 * the frame, the block loop and the entropy stage; the match finding of every block runs on the GPU.  Blocks are parsed
 * independently (no matches into earlier blocks).  Returns the number of records or ZSTD_SEQUENCE_PRODUCER_ERROR
 * ((size_t)-1): no device, dictSize != 0, level without a GPU parser (>= 13). */
ZSTDB200_API void* zstdb200_createSequenceProducerState(int device);
ZSTDB200_API void zstdb200_freeSequenceProducerState(void* state);
ZSTDB200_API size_t zstdb200_sequenceProducer(void* state, ZSTD_Sequence* outSeqs, size_t outSeqsCapacity, const void* src, size_t srcSize,
                                              const void* dict, size_t dictSize, int compressionLevel, size_t windowSize);

/* Device-memory calls (asynchronous on `stream`, a cudaStream_t passed as void*; 0 = the context's stream).
 * All pointers are device pointers; offsets are uint64 arrays of n+1 entries (item i = [off[i], off[i+1])).
 * compress_device writes frame i at d_slots + i*slotStride (slotStride >= ZSTD_compressBound(max chunk) + 32)
 * and its size / error code to d_frameSizes[i]; compact_device then scans the sizes and concatenates the
 * frames into d_out (coalesced), leaving the n+1 output offsets in d_outOffsets. */
ZSTDB200_API size_t zstdb200_compress_device(zstdb200_ctx* ctx, int level, size_t n, const void* d_src, const uint64_t* d_srcOffsets,
                                             void* d_slots, size_t slotStride, uint64_t* d_frameSizes, void* stream);
ZSTDB200_API size_t zstdb200_compact_device(zstdb200_ctx* ctx, size_t n, const void* d_slots, size_t slotStride, const uint64_t* d_frameSizes,
                                            void* d_out, uint64_t* d_outOffsets, void* stream);
/* compress_items_device compresses n items, item i = d_src[d_srcOffsets[i] .. d_srcOffsets[i+1]), each into the stream ZSTD_compress2
 * writes for it with ZSTDB200_c_multiFrame: one frame per chunkSize piece, each frame byte-identical to the reference's one-shot frame of
 * that piece at `level` and the context's frame options (checksum, content_size, magicless, explicit c_* parameters); an empty item is
 * the one empty frame.  The streams are packed in item order into d_dst: item i at [d_dstOffsets[i], d_dstOffsets[i+1]) (n+1 entries),
 * d_results[i] its size or the first error code among its frames.  The items are cut, compressed and packed on the GPU; nothing in the
 * call waits on the host.
 *   - chunkSize 0 or above 131072: parameter_outOfBound; a level without a GPU parser: parameter_unsupported (both returned, nothing queued).
 *   - dstCapacity must reach the sum, over every item's chunks, of ZSTD_compressBound(chunk), as for zstdb200_compress_chunks; when it
 *     does not, every item reports dstSize_tooSmall, every offset is 0 and nothing is compressed.
 *   - a frame the GPU does not serve (an optimal level on a chunk over 64 KB, levels 11-12 on a chunk of at most 16 KB) reports
 *     parameter_unsupported, and so does its item; the other items are unaffected.
 * The chunks are compressed in parts of P = min(16384, n + dstCapacity / chunkSize) by a CUDA graph the context keeps (built on the
 * first call and again when P, the level, chunkSize or a compression option changes); its workspace -- about 0.65 MB per part slot at
 * chunkSize 131072, the sequence records and the frame slots, and 40 bytes per item -- is kept too.  When the workspace or the graph
 * cannot be had the call returns memory_allocation and leaves neither the CUDA error state nor zstdb200_last_error() a trace.  The call
 * uses the context's work set 0 and must not overlap another call on it.
 * With option "seek_table" 1 each item is followed by its seek table (zstd's seekable format): a skippable frame of magic 0x184D2A5E
 * holding one entry per frame -- its compressed size, its regenerated size, and when the "checksum" option is on the frame's content
 * checksum (the descriptor's checksum flag is then set) -- then the frame count, the descriptor and 0x8F92EAB1.  The frames are the same
 * bytes as with the option off; item i is the option-off stream followed by its table, and d_results[i] and d_dstOffsets count the table.
 *   - dstCapacity must also reach 8 + E * k_i + 9 more bytes per item of k_i chunks (E = 12 with checksums, else 8); one byte short
 *     gives dstSize_tooSmall for every item as above.
 *   - an item of more than 0x8000000 chunks reports frameIndex_tooLarge; the other items are unaffected.  An item that fails has no table.
 *   - together with "magicless" the call returns parameter_unsupported and queues nothing.
 * The table's bookkeeping adds 8 bytes of kept workspace per chunk the capacity could hold. */
ZSTDB200_API size_t zstdb200_compress_items_device(zstdb200_ctx* ctx, int level, size_t chunkSize, size_t n, const void* d_src,
                                                   const uint64_t* d_srcOffsets, void* d_dst, size_t dstCapacity, uint64_t* d_dstOffsets,
                                                   uint64_t* d_results, void* stream);
/* decompress_device regenerates item i into d_dst + d_dstOffsets[i] (capacity d_dstOffsets[i+1] - d_dstOffsets[i]) and writes its size or
 * error code to d_results[i].  With dec_pipeline on (the default) the items are routed on the GPU: single-block frames with a content size
 * go to the staged decoder; items of several frames that are all one block are cut into their frames on the GPU, by the rule the
 * host-memory calls follow (every frame but the last declares its content size, at least 32 KB regenerated per frame on average), and
 * a CUDA graph runs the staged decoder over those frames in parts of 512 to 16384 (n); other items that are a whole number of frames with
 * a frame of several blocks or several frames (windows <= 2^27, skippable frames allowed, content sizes optional) go to a segment loop
 * that a CUDA graph drives on the GPU over the blocks of all of them when they are long or few -- many short ones decode faster one
 * warp each -- and everything else to the fused kernel, which also decodes again whole every item the loop doubts and every split item
 * whose frames do not each regenerate their declared size; results are those of the fused
 * decoder.  Nothing in the call waits on the host.  The loop's workspace (about 1.2 MB per dec_segment_blocks block, 600 MB at the
 * default) is allocated on the context's first such call and kept; when it or the graph cannot be had the call routes without the loop.
 * The split's list (about 52 bytes per entry, 2^16 + 16 n entries) is kept likewise; when it or its graph cannot be had no item is split.
 * The call uses the context's work set 0 and must not overlap another call on it.  zstdb200_segment_frames and zstdb200_split_items
 * do not count device calls. */
ZSTDB200_API size_t zstdb200_decompress_device(zstdb200_ctx* ctx, size_t n, const void* d_src, const uint64_t* d_srcOffsets,
                                               void* d_dst, const uint64_t* d_dstOffsets, uint64_t* d_results, void* stream);
/* decompress_bound_device finds on the GPU the room every item needs, from its frames alone.  d_bounds[i] (d_bounds may be NULL) is
 * ZSTD_decompressBound of item i = d_src[d_srcOffsets[i] .. d_srcOffsets[i+1]): the sum over its frames of the declared content size, or
 * the frame's blocks times its largest block size for a frame that declares none; skippable frames count 0; ZSTD_CONTENTSIZE_ERROR for
 * an item that is not a whole number of frames whose headers are valid.  On a magicless context the frames are ZSTD_f_zstd1_magicless
 * frames, and there are no skippable ones.  Item i's room is its bound, or 0 when the bound is ZSTD_CONTENTSIZE_ERROR; d_dstOffsets
 * (n+1 entries) is the exclusive scan of the rooms, the sum saturating at 2^64-1.  Nothing in the call waits on the host.
 *   - n above 2^31-1: srcSize_wrong (returned, nothing queued); n == 0 writes d_dstOffsets[0] = 0.
 *   - with d_bounds NULL the bounds go to a workspace the context keeps (8 bytes per item); when it cannot be had the call returns
 *     memory_allocation and leaves neither the CUDA error state nor zstdb200_last_error() a trace.
 * The call uses the context's work set 0 and must not overlap another call on it. */
ZSTDB200_API size_t zstdb200_decompress_bound_device(zstdb200_ctx* ctx, size_t n, const void* d_src, const uint64_t* d_srcOffsets,
                                                     uint64_t* d_dstOffsets, uint64_t* d_bounds, void* stream);
/* decompress_items_device regenerates items whose sizes only their frames know.  It writes d_dstOffsets as decompress_bound_device does,
 * then checks d_dstOffsets[n] <= dstCapacity on the GPU.
 *   - When the rooms fit, it decodes as zstdb200_decompress_device with those offsets: item i into d_dst + d_dstOffsets[i], d_results[i]
 *     its size or error code, each the same as zstdb200_decompress_device gives for these rooms.  The output is packed exactly when every
 *     frame declares its content size (the frames this library writes, and the reference's one-shot frames); otherwise the rooms are
 *     bounds, and d_results[i] says how much of item i's room was regenerated.
 *   - When they do not fit, every item reports dstSize_tooSmall and nothing is written to d_dst.  d_dstOffsets still holds the plan: a
 *     caller can read d_dstOffsets[n], allocate that much and call again.
 *   - n above 2^31-1: srcSize_wrong (returned, nothing queued); n == 0 writes d_dstOffsets[0] = 0.
 * With dec_pipeline 0 the plan is the same and the fused kernel decodes.  Nothing in the call waits on the host.  Besides
 * zstdb200_decompress_device's workspaces, the call keeps 24 bytes per item; when that cannot be had it returns memory_allocation and
 * leaves neither the CUDA error state nor zstdb200_last_error() a trace.  The call uses the context's work set 0 and must not overlap
 * another call on it. */
ZSTDB200_API size_t zstdb200_decompress_items_device(zstdb200_ctx* ctx, size_t n, const void* d_src, const uint64_t* d_srcOffsets, void* d_dst,
                                                     size_t dstCapacity, uint64_t* d_dstOffsets, uint64_t* d_results, void* stream);
/* decompress_ranges_device regenerates byte ranges of items, decoding only the frames that hold them.  Item i is
 * d_src[d_srcOffsets[i] .. d_srcOffsets[i+1]) (n+1 offsets).  Request r (m of them) asks for the regenerated bytes
 * [d_rangeBegins[r], d_rangeBegins[r] + len_r) of item d_rangeItems[r], len_r = d_dstOffsets[r+1] - d_dstOffsets[r] (m+1 offsets); they
 * go to d_dst + d_dstOffsets[r], and d_results[r] receives the number of bytes written or an error code.
 *   - Only the frames that regenerate at least one byte of a range are decoded.  The frames before it are walked (their headers and block
 *     headers), not decoded; the frames after it are not read.  A damaged frame outside a range does not affect that request.
 *   - Every frame covered is decoded whole and its checksum, if any, verified.  It must regenerate exactly its declared size, else the
 *     result is corruption_detected; its decode error is the one zstdb200_decompress_device gives for that frame alone in a room of its declared size.
 *   - When the item's content ends before the range does, the result is the bytes up to its end (as pread); a range starting at or past
 *     the end gives 0.  Bytes of the request's output beyond a short read are not written.
 *   - Every zstd frame the walk passes before the range's end must declare its content size, else the request gives
 *     parameter_unsupported.  Skippable frames and empty frames are walked and count 0.
 *   - A frame the range covers only in part must declare at most 131072 bytes (every frame compress_items_device, compress_chunks and the
 *     reference's one-shot path write does), else parameter_unsupported.  Frames of any size covered wholly decode straight into d_dst.
 *   - An item that cannot be walked as far as the range reaches gives the error ZSTD_findFrameCompressedSize gives for the first frame
 *     it cannot pass.  Where several failures apply, the first in item order wins.
 *   - d_rangeItems[r] >= n gives parameter_outOfBound; len_r == 0 gives 0 and reads nothing.
 *   - A failed request's output is unspecified, but nothing is ever written outside [d_dstOffsets[r], d_dstOffsets[r+1]).
 *   - m or n above 2^31-1: srcSize_wrong (returned, nothing queued); m == 0 queues nothing.
 * On a magicless context the items are ZSTD_f_zstd1_magicless frames, with no skippable frames.  With dec_pipeline 0 the plan is the
 * same and the fused kernel decodes.  Nothing in the call waits on the host.  The covered frames are decoded in parts of
 * P = min(16384, max(512, m)) frames, at most P / 2 of them covered in part, by a CUDA graph the context keeps (built on the first call
 * and again when P or a decoding option changes).  Its workspace does not grow with the ranges' lengths or frame counts: 64 bytes per
 * request, P / 2 scratch slots of 128 KB (32 MB at P = 512, 1 GB at P = 16384), 89 bytes per part slot, and the decoders' workspace for
 * P frames, which zstdb200_decompress_device's decode list shares.  When any of it cannot be had the call returns memory_allocation and
 * leaves neither the CUDA error state nor zstdb200_last_error() a trace.  The call uses the context's work set 0 and must not overlap
 * another call on it.
 * With option "seek_table" 1 a request whose item ends with a valid seek table is located through it, without walking the frames before
 * the range.  Valid: the item is at least 17 bytes and ends with 0x8F92EAB1, the descriptor's reserved bits (6-2) are 0, the frame count
 * k is at most 0x8000000, the table (8 + E k + 9 bytes) fits the item and starts with 0x184D2A5E and E k + 9, and the entries'
 * compressed sizes sum to exactly the bytes before it.  Any other item is walked as with the option off, with the same results.
 * Through a table:
 *   - entries of regenerated size 0 are passed; an entry that holds a byte of the range is decoded, and frames need not declare their
 *     content size.  An entry covered in part must regenerate at most 131072 bytes, else parameter_unsupported.
 *   - each decoded entry's frame must be walkable (else ZSTD_findFrameCompressedSize's error), not skippable, of the entry's compressed
 *     size and, if it declares a content size, of the entry's regenerated size (else corruption_detected); it must regenerate exactly
 *     that size, with the error rule above; and with the table's checksum flag its bytes must hash to the entry's checksum (the low 32
 *     bits of XXH64), else checksum_wrong.  The first failure in item order still wins.
 *   - the content ends at the sum of the entries' regenerated sizes; short reads and ranges past the end are as above.
 *   - together with "magicless" the call returns parameter_unsupported and queues nothing.
 * The workspace is the same; the graph is built again when the option changes. */
ZSTDB200_API size_t zstdb200_decompress_ranges_device(zstdb200_ctx* ctx, size_t n, const void* d_src, const uint64_t* d_srcOffsets,
                                                      size_t m, const uint64_t* d_rangeItems, const uint64_t* d_rangeBegins,
                                                      void* d_dst, const uint64_t* d_dstOffsets, uint64_t* d_results, void* stream);
ZSTDB200_API size_t zstdb200_sync(zstdb200_ctx* ctx, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* ZSTDB200_H */
