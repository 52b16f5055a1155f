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
/* tuning knobs (also read from the environment at context creation):
 *   "enc_warps_per_sm" / ZSTDB200_ENC_WARPS_PER_SM, "dec_warps_per_sm" / ZSTDB200_DEC_WARPS_PER_SM,
 *   "parse_lanes" (4|8|16|32), "parse_blocks_per_sm", "lazy_blocks_per_sm" (4|6|8: residency of the levels >= 5 parse kernel),
 *   "parse_est_bytes" (prefix parsed for the cost estimate that orders the parse), "dec_pipeline" (0|1),
 *   "host_slices" / "host_slices_dec" (slices of the synchronous host-memory calls; defaults 1 / 2), "timing" (0|1),
 *   "entropy_overlap" (0|1, default 1 / ZSTDB200_ENTROPY_OVERLAP: the entropy stage is launched as a programmatic dependent of the parse and
 *   takes frames in the order their parse finishes, filling the SMs the parse's tail leaves idle),
 *   "kernel_fifo" (0|1, default 1 / ZSTDB200_KERNEL_FIFO: the kernel sections of host-memory operations queued on different work sets run
 *   one after the other in submission order -- copies still overlap them; two batches in the kernels at once only slow each other down) */
ZSTDB200_API int zstdb200_set_option(zstdb200_ctx* ctx, const char* name, long long value);
ZSTDB200_API unsigned long long zstdb200_kernel_launches(const zstdb200_ctx* ctx);   /* kernels launched so far */
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
ZSTDB200_API size_t zstdb200_decompress_device(zstdb200_ctx* ctx, size_t n, const void* d_src, const uint64_t* d_srcOffsets,
                                               void* d_dst, const uint64_t* d_dstOffsets, uint64_t* d_results, void* stream);
ZSTDB200_API size_t zstdb200_sync(zstdb200_ctx* ctx, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* ZSTDB200_H */
