// zb_libzstd.cpp -- the libzstd-compatible entry points (ZSTD_*) of include/zstdb200.h, host code on the batch API: every
// (de)compression takes a pooled batch context, configures it through zstdb200_set_option alone and hands it the work.
#include <cuda_runtime_api.h>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <new>
#include <vector>

#include "../../include/zstdb200.h"
#include "zb_decode.cuh"
#include "zb_encode.cuh"

using namespace zb;

static_assert(ZSTD_c_strategy - ZSTD_c_windowLog + 1 == sizeof CPARAM_BOUNDS / sizeof CPARAM_BOUNDS[0], "CPARAM_BOUNDS is indexed by ZSTD_cParameter");

namespace {

struct PoolEntry { int device; zstdb200_ctx* c; };
std::mutex g_poolMutex;
std::vector<PoolEntry> g_pool;     // idle contexts, any device; a caller gets one of its current device

// A batch context taken from the pool for one call on the caller's current device.  Its whole configuration is set on
// acquire -- the flags (FRAME_*) of the frames it writes or reads and every explicit compression parameter, zeros
// included -- so nothing of an earlier call carries over.  ok: a context was made and took every option.
struct PooledCtx {
    int device = 0; zstdb200_ctx* c = nullptr; bool ok = false;
    PooledCtx(u32 flags, const CParams& ov) {
        if (cudaGetDevice(&device) != cudaSuccess) { (void)cudaGetLastError(); device = -1; }
        {   std::lock_guard<std::mutex> lk(g_poolMutex);
            for (size_t k = g_pool.size(); k-- > 0;)
                if (g_pool[k].device == device) { c = g_pool[k].c; g_pool.erase(g_pool.begin() + (ptrdiff_t)k); break; } }
        if (!c && !(c = zstdb200_create(device))) return;
        int rc = zstdb200_set_option(c, "checksum", (flags & FRAME_CHECKSUM) != 0) | zstdb200_set_option(c, "content_size", !(flags & FRAME_NO_CONTENT_SIZE)) |
                 zstdb200_set_option(c, "magicless", (flags & FRAME_MAGICLESS) != 0);
        for (auto const& b : CPARAM_BOUNDS) rc |= zstdb200_set_option(c, b.option, ov.*(b.member));
        ok = rc == 0;
    }
    ~PooledCtx() { if (c) { std::lock_guard<std::mutex> lk(g_poolMutex); g_pool.push_back({ device, c }); } }
};

// host-side frame walks (no GPU needed): same parsers as the kernels, host instantiation of the headers
// `missing` (optional): when the frame is cut short (srcSize_wrong), the least number of further bytes that lets the walk advance;
// *nbBlocks then holds the whole blocks present
size_t host_find_frame_size(const u8* src, size_t srcSize, size_t* nbBlocks, FrameHeader* fhOut, u32 magicless = 0, size_t* missing = nullptr) {
    if (missing) *missing = 1;
    // inputs may be unaligned / tiny: copy the few bytes we look at into an aligned scratch when needed
    FrameHeader fh;
    size_t const hn = srcSize < 18 ? srcSize : 18;
    alignas(8) u8 buf[64] = {0};
    memcpy(buf + 8, src, hn);
    size_t const r = read_frame_header(&fh, buf + 8, hn, magicless);
    if (isErr(r)) return r;
    if (r > 0) { if (missing) *missing = r > srcSize ? r - srcSize : 1; return ERR(E_srcSize_wrong); }
    if (fhOut) *fhOut = fh;
    if (fh.skippable) { if ((u64)fh.skipLen + 8 > srcSize) { if (missing) *missing = (size_t)((u64)fh.skipLen + 8 - srcSize); return ERR(E_srcSize_wrong); } if (nbBlocks) *nbBlocks = 0; return 8 + (size_t)fh.skipLen; }
    size_t pos = fh.headerSize, blocks = 0;
    for (;;) {
        if (nbBlocks) *nbBlocks = blocks;
        if (srcSize - pos < 3) { if (missing) *missing = 3 - (srcSize - pos); return ERR(E_srcSize_wrong); }
        u32 const bh = (u32)src[pos] | ((u32)src[pos + 1] << 8) | ((u32)src[pos + 2] << 16);
        u32 const type = (bh >> 1) & 3; size_t cSize = bh >> 3;
        if (type == 3) return ERR(E_corruption_detected);
        if (type == 1) cSize = 1;
        if (3 + cSize > srcSize - pos) { if (missing) *missing = 3 + cSize - (srcSize - pos) + ((bh & 1) ? (fh.checksum ? 4 : 0) : 3); return ERR(E_srcSize_wrong); }
        pos += 3 + cSize; blocks++;
        if (bh & 1) break;
    }
    if (fh.checksum) { if (srcSize - pos < 4) { if (missing) *missing = 4 - (srcSize - pos); return ERR(E_srcSize_wrong); } pos += 4; }
    if (nbBlocks) *nbBlocks = blocks;
    return pos;
}

const char* error_string(int code) {
    switch (code) {
    case 0: return "No error detected";
    case 1: return "Error (generic)";
    case 10: return "Unknown frame descriptor";
    case 12: return "Version not supported";
    case 14: return "Unsupported frame parameter";
    case 16: return "Frame requires too much memory for decoding";
    case 20: return "Data corruption detected";
    case 22: return "Restored data doesn't match checksum";
    case 24: return "Header of Literals' block doesn't respect format specification";
    case 30: return "Dictionary is corrupted";
    case 32: return "Dictionary mismatch";
    case 34: return "Cannot create Dictionary from provided samples";
    case 40: return "Unsupported parameter";
    case 41: return "Unsupported combination of parameters";
    case 42: return "Parameter is out of bound";
    case 44: return "tableLog requires too much memory : unsupported";
    case 46: return "Unsupported max Symbol Value : too large";
    case 48: return "Specified maxSymbolValue is too small";
    case 49: return "This mode cannot generate an uncompressed block";
    case 50: return "pledged buffer stability condition is not respected";
    case 60: return "Operation not authorized at current processing stage";
    case 62: return "Context should be init first";
    case 64: return "Allocation error : not enough memory";
    case 66: return "workSpace buffer is not large enough";
    case 70: return "Destination buffer is too small";
    case 72: return "Src size is incorrect";
    case 74: return "Operation on NULL destination buffer";
    case 80: return "Operation made no progress over multiple calls, due to output buffer being full";
    case 82: return "Operation made no progress over multiple calls, due to input being empty";
    case 100: return "Frame index is too large";
    case 102: return "An I/O error occurred when reading/seeking";
    case 104: return "Destination buffer is wrong";
    case 105: return "Source buffer is wrong";
    case 106: return "Block-level external sequence producer returned an error code";
    case 107: return "External sequences are not valid";
    default: return "Unspecified error code";
    }
}

}  // namespace

// byte buffer of the streaming layer: grows without zero-filling (a std::vector would memset a GiB per batch)
struct RawBuf {
    u8* p = nullptr; size_t n = 0, cap = 0;
    ~RawBuf() { free(p); }
    RawBuf() = default; RawBuf(const RawBuf&) = delete; RawBuf& operator=(const RawBuf&) = delete;
    size_t size() const { return n; }
    bool empty() const { return n == 0; }
    u8* data() { return p; }
    void clear() { n = 0; }
    void resize(size_t want) {      // throws std::bad_alloc like a vector would; contents up to min(n, want) are kept
        if (want > cap) { size_t c = cap ? cap : 4096; while (c < want) c += c / 2 + 4096; u8* q = (u8*)realloc(p, c); if (!q) throw std::bad_alloc(); p = q; cap = c; }
        n = want;
    }
    void append(const u8* src, size_t k) { size_t const at = n; resize(n + k); if (k) memcpy(p + at, src, k); }
    void erase_front(size_t k) { if (k >= n) { n = 0; return; } memmove(p, p + k, n - k); n -= k; }
    void assign(const u8* src, size_t k) { n = 0; append(src, k); }
};

struct ZSTD_CCtx_s {
    int level = 3;
    int checksum = 0, contentSize = 1, dictID = 1, format = 0;      // format: ZSTD_f_zstd1 = 0, ZSTD_f_zstd1_magicless = 1
    u32 frameFlags() const { return (checksum ? FRAME_CHECKSUM : 0u) | (contentSize ? 0u : FRAME_NO_CONTENT_SIZE) | (format ? FRAME_MAGICLESS : 0u); }
    unsigned long long ingested = 0, consumed = 0, produced = 0, flushed = 0;      // ZSTD_getFrameProgression
    CParams ov = { 0, 0, 0, 0, 0, 0, 0 };      // ZSTD_c_windowLog ... ZSTD_c_strategy, 0 = from the level (J/ZstdCompressCtx.setWindowLog ... setStrategy)
    bool unsupportedParam = false;
    bool foreignProducer = false;      // ZSTD_registerSequenceProducer with a non-NULL function
    bool multiFrame = getenv("ZSTDB200_MULTIFRAME") && atoi(getenv("ZSTDB200_MULTIFRAME")) != 0;   // see ZSTDB200_c_multiFrame
    // streaming state
    RawBuf inBuf;               // pending input (< one block)
    RawBuf outBuf;              // produced frames not yet handed out
    size_t outPos = 0;
    bool emittedAny = false;    // a frame went out since the last reset / end of stream
};
struct ZSTD_DCtx_s {
    int format = 0;             // ZSTD_d_format
    u64 maxWindowSize = (1ull << 27) + 1;      // ZSTD_d_windowLogMax (default ZSTD_WINDOWLOG_LIMIT_DEFAULT, N/decompress/zstd_decompress.c:249), enforced by ZSTD_decompressStream like the reference (:2227-2228)
    RawBuf inBuf;               // bytes of the frame being collected
    RawBuf outBuf;              // regenerated bytes not yet handed out
    size_t outPos = 0;
    zstdb200_fstream* fs = nullptr;      // a frame of more blocks than one segment, streamed segment by segment
    u32 segBlocks = 0;                   // blocks per segment of the batch contexts (0: not asked yet)
    void end_frame_stream() { zstdb200_fstream_free(fs); fs = nullptr; }
    ~ZSTD_DCtx_s() { end_frame_stream(); }
};

extern "C" {

unsigned ZSTD_isError(size_t code) { return isErr(code); }
int ZSTD_getErrorCode(size_t code) { return isErr(code) ? (int)(0 - code) : 0; }
const char* ZSTD_getErrorName(size_t code) { return error_string(ZSTD_getErrorCode(code)); }
unsigned ZSTD_versionNumber(void) { return 10507; }
const char* ZSTD_versionString(void) { return "1.5.7"; }
int ZSTD_minCLevel(void) { return -(1 << 17); }
int ZSTD_maxCLevel(void) { return 22; }
int ZSTD_defaultCLevel(void) { return 3; }
size_t ZSTD_compressBound(size_t srcSize) { return compress_bound(srcSize); }

ZSTD_CCtx* ZSTD_createCCtx(void) { return new (std::nothrow) ZSTD_CCtx_s(); }
size_t ZSTD_freeCCtx(ZSTD_CCtx* c) { delete c; return 0; }
ZSTD_DCtx* ZSTD_createDCtx(void) { return new (std::nothrow) ZSTD_DCtx_s(); }
size_t ZSTD_freeDCtx(ZSTD_DCtx* d) { delete d; return 0; }

size_t ZSTD_CCtx_setParameter(ZSTD_CCtx* c, ZSTD_cParameter param, int value) {
    if (!c) return ERR(E_GENERIC);
    switch (param) {
    case ZSTD_c_compressionLevel:
        if (value > 22) value = 22;
        if (value < -(1 << 17)) value = -(1 << 17);
        c->level = value ? value : 3;
        return (size_t)(value > 0 ? value : 0);
    case ZSTD_c_checksumFlag: c->checksum = value != 0; return (size_t)c->checksum;
    case ZSTD_c_contentSizeFlag: c->contentSize = value != 0; return (size_t)c->contentSize;
    case ZSTD_c_dictIDFlag: c->dictID = value != 0; return (size_t)c->dictID;
    case ZSTD_c_format:          // N/jni_zstd.c:362-363 (setCompressionMagicless), J/ZstdCompressCtx.setMagicless
        if (value != 0 && value != 1) return ERR(E_parameter_outOfBound);
        c->format = value; return (size_t)value;
    case ZSTD_c_nbWorkers: if (value != 0) c->unsupportedParam = true; return (size_t)value;
    case ZSTDB200_c_multiFrame: c->multiFrame = value != 0; return (size_t)c->multiFrame;
    // explicit compression parameters (N/jni_zstd.c setCompressionWindowLog ... setCompressionStrategy, N/jni_fast_zstd.c): applied over
    // the level's row like ZSTD_getCParamsFromCCtxParams does; bounds of ZSTD_cParam_getBounds (N/compress/zstd_compress.c:420-520)
    case ZSTD_c_windowLog: case ZSTD_c_hashLog: case ZSTD_c_chainLog: case ZSTD_c_searchLog: case ZSTD_c_minMatch: case ZSTD_c_targetLength: case ZSTD_c_strategy: {
        CParamBound const& b = CPARAM_BOUNDS[param - ZSTD_c_windowLog];
        if (!b.accepts(value)) return ERR(E_parameter_outOfBound);
        c->ov.*(b.member) = (u32)value; return (size_t)value; }
    default:
        // anything else that would change the emitted bytes (LDM, workers, block splitter ...) is not reproduced by this
        // build => the next compression call reports parameter_unsupported
        if (value != 0) c->unsupportedParam = true;
        return (size_t)value;
    }
}
size_t ZSTD_CCtx_reset(ZSTD_CCtx* c, ZSTD_ResetDirective reset) {
    if (!c) return ERR(E_GENERIC);
    if (reset == ZSTD_reset_session_only || reset == ZSTD_reset_session_and_parameters) { c->inBuf.clear(); c->outBuf.clear(); c->outPos = 0; c->emittedAny = false;
                                                                                         c->ingested = c->consumed = c->produced = c->flushed = 0; }
    if (reset == ZSTD_reset_parameters || reset == ZSTD_reset_session_and_parameters) { c->level = 3; c->checksum = 0; c->contentSize = 1; c->dictID = 1; c->format = 0; c->unsupportedParam = false; c->foreignProducer = false; c->ov = CParams{ 0, 0, 0, 0, 0, 0, 0 }; }
    return 0;
}
size_t ZSTD_DCtx_reset(ZSTD_DCtx* d, ZSTD_ResetDirective reset) {
    if (!d) return ERR(E_GENERIC);
    if (reset != ZSTD_reset_parameters) { d->inBuf.clear(); d->outBuf.clear(); d->outPos = 0; d->end_frame_stream(); }
    if (reset != ZSTD_reset_session_only) { d->format = 0; d->maxWindowSize = (1ull << 27) + 1; }
    return 0;
}
// N/jni_zstd.c:403 (setDecompressionLongMax), :413-414 (setDecompressionMagicless); ZSTD_dParam_getBounds, N/decompress/zstd_decompress.c:1838-1878
size_t ZSTD_DCtx_setParameter(ZSTD_DCtx* d, ZSTD_dParameter param, int value) {
    if (!d) return ERR(E_GENERIC);
    if (!d->inBuf.empty() || d->outPos < d->outBuf.size() || d->fs) return ERR(E_stage_wrong);
    switch (param) {
    case ZSTD_d_windowLogMax:
        if (value == 0) value = 27;
        if (value < 10 || value > 31) return ERR(E_parameter_outOfBound);
        d->maxWindowSize = 1ull << value; return 0;
    case ZSTD_d_format:
        if (value != 0 && value != 1) return ERR(E_parameter_outOfBound);
        d->format = value; return 0;
    default: return ERR(E_parameter_unsupported);
    }
}
size_t ZSTD_CCtx_setPledgedSrcSize(ZSTD_CCtx* c, unsigned long long) { return c ? 0 : ERR(E_GENERIC); }

// ---- context-taking entry points of features that are NOT built (dictionaries, foreign sequence producers).  The JNI glue calls
// them with contexts created by ZSTD_createCCtx / ZSTD_createDCtx of THIS library (N/jni_zstd.c:271-346, N/jni_fast_zstd.c:325-362,673-710,
// :133-250); if they resolved to a CPU libzstd linked behind for the cold path, that library would reinterpret our context objects.
// So they live here and refuse loudly; clearing calls (NULL / empty dictionary) succeed like in the reference.
size_t ZSTD_CCtx_loadDictionary(ZSTD_CCtx* c, const void* dict, size_t dictSize) { if (!c) return ERR(E_GENERIC); return (dict && dictSize) ? ERR(E_parameter_unsupported) : 0; }
size_t ZSTD_CCtx_refCDict(ZSTD_CCtx* c, const ZSTD_CDict* cdict) { if (!c) return ERR(E_GENERIC); return cdict ? ERR(E_parameter_unsupported) : 0; }
size_t ZSTD_DCtx_loadDictionary(ZSTD_DCtx* d, const void* dict, size_t dictSize) { if (!d) return ERR(E_GENERIC); return (dict && dictSize) ? ERR(E_parameter_unsupported) : 0; }
size_t ZSTD_DCtx_refDDict(ZSTD_DCtx* d, const ZSTD_DDict* ddict) { if (!d) return ERR(E_GENERIC); return ddict ? ERR(E_parameter_unsupported) : 0; }
size_t ZSTD_compress_usingCDict(ZSTD_CCtx* c, void*, size_t, const void*, size_t, const ZSTD_CDict*) { return c ? ERR(E_parameter_unsupported) : ERR(E_GENERIC); }
// an external sequence producer would replace the GPU match finder: registering one makes the next compression report parameter_unsupported
// (the reverse direction -- this library AS the producer of a CPU libzstd -- is zstdb200_sequenceProducer)
void ZSTD_registerSequenceProducer(ZSTD_CCtx* c, void* state, ZSTD_sequenceProducer_F fn) { (void)state; if (c) c->foreignProducer = fn != nullptr; }

// Every compression: checks the parameters, then compresses through a pooled context configured with the frame flags and the
// explicit parameters `ov` -- `src` (at most one block) as one frame, or with perBlock as one independent frame per block.
// Returns the bytes written to dst or an error code.
static size_t compress_pooled(int level, u32 flags, const CParams& ov, bool unsupported, bool perBlock, void* dst, size_t dstCapacity,
                              const void* src, size_t srcSize) {
    if (unsupported) return ERR(E_parameter_unsupported);
    {   CParams cp; if (!get_cparams(&cp, level, srcSize < BLOCKSIZE_MAX ? srcSize : BLOCKSIZE_MAX, ov.any_set() ? &ov : nullptr)) return ERR(E_parameter_unsupported); }
    PooledCtx g(flags, ov);
    if (!g.ok) return ERR(E_GENERIC);
    size_t total = 0;
    size_t const r = perBlock ? zstdb200_compress_chunks(g.c, level, src, srcSize, BLOCKSIZE_MAX, dst, dstCapacity, nullptr, &total)
                              : zstdb200_compress_batch(g.c, level, 1, &src, &srcSize, &dst, &dstCapacity, &total);
    return isErr(r) ? r : total;
}
static size_t compress_one(int level, u32 flags, bool unsupported, void* dst, size_t dstCapacity, const void* src, size_t srcSize,
                           bool multiFrame = false, const CParams& ov = CParams{}) {
    // A multi-block frame (cross-block window, repeat modes) is serial and outside this build's bit-exact scope.  Only on
    // request the input is written as one independent frame per 128 KB -- a legal zstd stream for every decoder, but
    // not the reference's bytes.
    if (srcSize > BLOCKSIZE_MAX && !multiFrame) return ERR(E_parameter_unsupported);
    return compress_pooled(level, flags, ov, unsupported, srcSize > BLOCKSIZE_MAX, dst, dstCapacity, src, srcSize);
}
size_t ZSTD_compress2(ZSTD_CCtx* c, void* dst, size_t dstCapacity, const void* src, size_t srcSize) {
    if (!c) return ERR(E_GENERIC);
    return compress_one(c->level, c->frameFlags(), c->unsupportedParam || c->foreignProducer, dst, dstCapacity, src, srcSize, c->multiFrame, c->ov);
}
size_t ZSTD_compressCCtx(ZSTD_CCtx*, void* dst, size_t dstCapacity, const void* src, size_t srcSize, int level) {
    return compress_one(level ? level : 3, 0, false, dst, dstCapacity, src, srcSize);
}
size_t ZSTD_compress(void* dst, size_t dstCapacity, const void* src, size_t srcSize, int level) {
    return compress_one(level ? level : 3, 0, false, dst, dstCapacity, src, srcSize);
}
static size_t decompress_one(void* dst, size_t dstCapacity, const void* src, size_t srcSize, int format);
size_t ZSTD_decompressDCtx(ZSTD_DCtx* d, void* dst, size_t dstCapacity, const void* src, size_t srcSize) {
    return decompress_one(dst, dstCapacity, src, srcSize, d ? d->format : 0);
}
size_t ZSTD_decompress(void* dst, size_t dstCapacity, const void* src, size_t srcSize) { return decompress_one(dst, dstCapacity, src, srcSize, 0); }
size_t ZSTD_decompress_usingDDict(ZSTD_DCtx* d, void* dst, size_t dstCapacity, const void* src, size_t srcSize, const ZSTD_DDict* ddict) {
    if (ddict) return ERR(E_parameter_unsupported);          // a NULL DDict means "no dictionary" (N/decompress/zstd_decompress.c:1689-1696)
    return decompress_one(dst, dstCapacity, src, srcSize, d ? d->format : 0);
}
static size_t decompress_one(void* dst, size_t dstCapacity, const void* src, size_t srcSize, int format) {
    if (srcSize == 0) return 0;
    PooledCtx g(format ? FRAME_MAGICLESS : 0u, CParams{});
    if (!g.ok) return ERR(E_GENERIC);
    size_t out = 0;
    size_t const r = zstdb200_decompress_batch(g.c, 1, &src, &srcSize, &dst, &dstCapacity, &out);
    return isErr(r) ? r : out;
}

// ZSTD_getFrameHeader_advanced (N/decompress/zstd_decompress.c:447-551; N/jni_zstd.c:35 for magicless sizes): host-side parse
size_t ZSTD_getFrameHeader_advanced(ZSTD_FrameHeader* zfh, const void* src, size_t srcSize, ZSTD_format_e format) {
    if (!zfh || (srcSize > 0 && !src)) return ERR(E_GENERIC);
    FrameHeader fh; alignas(8) u8 buf[64] = {0};
    size_t const hn = srcSize < 18 ? srcSize : 18;
    if (hn) memcpy(buf + 8, src, hn);
    size_t const r = read_frame_header(&fh, buf + 8, hn, format == ZSTD_f_zstd1_magicless);
    if (r != 0) return r;
    memset(zfh, 0, sizeof *zfh);
    zfh->headerSize = fh.headerSize; zfh->dictID = fh.dictID;
    if (fh.skippable) { zfh->frameType = ZSTD_skippableFrame; zfh->frameContentSize = fh.skipLen; return 0; }
    zfh->frameType = ZSTD_frame;
    zfh->frameContentSize = fh.hasContentSize ? fh.contentSize : ZSTD_CONTENTSIZE_UNKNOWN;
    zfh->windowSize = fh.windowSize; zfh->blockSizeMax = fh.blockSizeMax; zfh->checksumFlag = fh.checksum;
    return 0;
}
size_t ZSTD_getFrameHeader(ZSTD_FrameHeader* zfh, const void* src, size_t srcSize) { return ZSTD_getFrameHeader_advanced(zfh, src, srcSize, ZSTD_f_zstd1); }
size_t ZSTD_frameHeaderSize(const void* src, size_t srcSize) {      // :432-435
    if (srcSize < 5) return ERR(E_srcSize_wrong);
    u32 const fhd = ((const u8*)src)[4], dictID = fhd & 3, single = (fhd >> 5) & 1, fcsID = fhd >> 6;
    return 5 + !single + (dictID == 3 ? 4 : dictID) + (fcsID == 0 ? 0 : (1u << fcsID)) + (single && !fcsID);
}
unsigned ZSTD_isFrame(const void* src, size_t srcSize) {            // :380-393 (no legacy formats)
    if (srcSize < 4) return 0;
    u32 m; memcpy(&m, src, 4);
    return m == MAGIC || (m & 0xFFFFFFF0u) == 0x184D2A50u;
}
unsigned ZSTD_isSkippableFrame(const void* src, size_t srcSize) {   // :402-409
    if (srcSize < 4) return 0;
    u32 m; memcpy(&m, src, 4);
    return (m & 0xFFFFFFF0u) == 0x184D2A50u;
}
unsigned ZSTD_getDictID_fromFrame(const void* src, size_t srcSize) {   // :1644-1650 (N/jni_zstd.c:139,156)
    ZSTD_FrameHeader zfh;
    size_t const r = ZSTD_getFrameHeader(&zfh, src, srcSize);
    return isErr(r) ? 0 : zfh.dictID;
}
unsigned long long ZSTD_getFrameContentSize(const void* src, size_t srcSize) {      // :643-658
    ZSTD_FrameHeader zfh;
    if (ZSTD_getFrameHeader(&zfh, src, srcSize) != 0) return ZSTD_CONTENTSIZE_ERROR;
    return zfh.frameType == ZSTD_skippableFrame ? 0 : zfh.frameContentSize;
}
// ZSTD_getFrameProgression (N/compress/zstd_compress.c:1898-1916; N/jni_fast_zstd.c:373, J/ZstdCompressCtx.getFrameProgression)
ZSTD_frameProgression ZSTD_getFrameProgression(const ZSTD_CCtx* c) {
    ZSTD_frameProgression fp; memset(&fp, 0, sizeof fp);
    if (c) { fp.ingested = c->ingested; fp.consumed = c->consumed; fp.produced = c->produced; fp.flushed = c->flushed; }
    return fp;
}
size_t ZSTD_findFrameCompressedSize(const void* src, size_t srcSize) { return host_find_frame_size((const u8*)src, srcSize, nullptr, nullptr); }
unsigned long long ZSTD_decompressBound(const void* srcv, size_t srcSize) {
    const u8* src = (const u8*)srcv; unsigned long long bound = 0;
    while (srcSize > 0) {
        size_t blocks = 0; FrameHeader fh;
        size_t const c = host_find_frame_size(src, srcSize, &blocks, &fh);
        if (isErr(c)) return ZSTD_CONTENTSIZE_ERROR;
        if (!fh.skippable) bound += fh.hasContentSize ? fh.contentSize : (unsigned long long)blocks * fh.blockSizeMax;
        src += c; srcSize -= c;
    }
    return bound;
}

// ---- streaming: independent-frames mode (see INTEGRATION.md)
ZSTD_CStream* ZSTD_createCStream(void) { return ZSTD_createCCtx(); }
size_t ZSTD_freeCStream(ZSTD_CStream* z) { return ZSTD_freeCCtx(z); }
size_t ZSTD_initCStream(ZSTD_CStream* z, int level) { if (!z) return ERR(E_GENERIC); ZSTD_CCtx_reset(z, ZSTD_reset_session_only); z->level = level ? level : 3; return 0; }
size_t ZSTD_CStreamInSize(void) { return BLOCKSIZE_MAX; }
size_t ZSTD_CStreamOutSize(void) { return compress_bound(BLOCKSIZE_MAX) + 3 + 4; }
size_t ZSTD_DStreamInSize(void) { return BLOCKSIZE_MAX + 3; }
size_t ZSTD_DStreamOutSize(void) { return BLOCKSIZE_MAX; }

// Streams are sequences of independent frames, one per 128 KB block (INTEGRATION.md section 1).  Both directions batch: whatever
// whole blocks / whole frames the caller offers in one call go through the batch kernels together -- a direct buffer of hundreds
// of MiB costs one copy-in, one chain of launches and one copy-out, not one per block (J/ZstdOutputStreamNoFinalizer.java:400-518
// and J/ZstdDirectBufferCompressingStreamNoFinalizer hand the whole remaining source to every call).
static size_t stream_batch_bytes() {        // input taken per batch; ZSTDB200_STREAM_BATCH_MB overrides (1 .. 4096)
    static size_t const v = [] { const char* e = getenv("ZSTDB200_STREAM_BATCH_MB"); long m = e ? atol(e) : 1024; if (m < 1) m = 1; if (m > 4096) m = 4096; return (size_t)m << 20; }();
    return v;
}
static size_t cstream_drain(ZSTD_CCtx* c, ZSTD_outBuffer* out) {
    size_t const avail = c->outBuf.size() - c->outPos, room = out->size - out->pos;
    size_t const k = avail < room ? avail : room;
    if (k) { memcpy((u8*)out->dst + out->pos, c->outBuf.data() + c->outPos, k); out->pos += k; c->outPos += k; c->flushed += k; }
    if (c->outPos == c->outBuf.size()) { c->outBuf.clear(); c->outPos = 0; }
    return c->outBuf.size() - c->outPos;
}
// n bytes at p -> frames of at most one block each: straight into the caller's buffer when the whole bound fits there, else
// appended to outBuf
static size_t cstream_emit(ZSTD_CCtx* c, const u8* p, size_t n, ZSTD_outBuffer* out = nullptr) {
    size_t const blocks = n ? (n + BLOCKSIZE_MAX - 1) / BLOCKSIZE_MAX : 1;
    size_t const one = compress_bound(BLOCKSIZE_MAX) < 18 ? 18 : compress_bound(BLOCKSIZE_MAX);
    size_t const bound = blocks * one;
    bool const direct = out && c->outBuf.empty() && out->size - out->pos >= bound;
    size_t const at = c->outBuf.size();
    if (!direct) c->outBuf.resize(at + bound);
    size_t const total = compress_pooled(c->level, c->frameFlags(), c->ov, c->unsupportedParam || c->foreignProducer, true,
                                         direct ? (u8*)out->dst + out->pos : c->outBuf.data() + at, bound, p, n);
    if (isErr(total)) { if (!direct) c->outBuf.resize(at); return total; }
    if (direct) { out->pos += total; c->flushed += total; } else c->outBuf.resize(at + total);
    c->consumed += n; c->produced += total; c->emittedAny = true;
    return 0;
}
static size_t compress_stream2(ZSTD_CCtx* c, ZSTD_outBuffer* out, ZSTD_inBuffer* in, ZSTD_EndDirective endOp) {
    if (!c || !out || !in) return ERR(E_GENERIC);
    if (out->pos > out->size) return ERR(E_dstSize_tooSmall);
    if (in->pos > in->size) return ERR(E_srcSize_wrong);
    // hand out what is pending first
    if (cstream_drain(c, out) > 0) return c->outBuf.size() - c->outPos;
    // 1. a partial block left over from earlier calls is filled up first
    if (!c->inBuf.empty() && in->pos < in->size) {
        size_t const want = BLOCKSIZE_MAX - c->inBuf.size();
        size_t const k = (in->size - in->pos) < want ? (in->size - in->pos) : want;
        c->inBuf.append((const u8*)in->src + in->pos, k);
        in->pos += k; c->ingested += k;
        if (c->inBuf.size() == BLOCKSIZE_MAX) { size_t const r = cstream_emit(c, c->inBuf.data(), c->inBuf.size(), out); if (isErr(r)) return r; c->inBuf.clear(); }
    }
    // 2. whole blocks straight from the caller's buffer, as many as one batch takes
    if (c->inBuf.empty() && c->outBuf.empty()) {
        size_t whole = (in->size - in->pos) / BLOCKSIZE_MAX * BLOCKSIZE_MAX;
        if (whole > stream_batch_bytes()) whole = stream_batch_bytes() / BLOCKSIZE_MAX * BLOCKSIZE_MAX;
        if (whole) {
            size_t const r = cstream_emit(c, (const u8*)in->src + in->pos, whole, out); if (isErr(r)) return r;
            in->pos += whole; c->ingested += whole;
        }
    }
    // 3. the tail shorter than a block waits for more input (or for flush / end)
    if (c->outBuf.empty() && in->pos < in->size && in->size - in->pos < BLOCKSIZE_MAX) {
        size_t const k = in->size - in->pos;
        c->inBuf.append((const u8*)in->src + in->pos, k);
        in->pos += k; c->ingested += k;
    }
    if (endOp != ZSTD_e_continue && in->pos == in->size) {
        // an empty stream still is one (empty) frame; a stream whose blocks all went out already needs nothing more
        if (!c->inBuf.empty() || (endOp == ZSTD_e_end && !c->emittedAny)) {
            size_t const r = cstream_emit(c, c->inBuf.data(), c->inBuf.size(), out); if (isErr(r)) return r;
            c->inBuf.clear();
        }
    }
    size_t const pending = cstream_drain(c, out);
    if (endOp == ZSTD_e_continue) return pending ? pending : (BLOCKSIZE_MAX - c->inBuf.size());
    if (in->pos < in->size) return pending ? pending : 1;      // more input to take: call again
    if (pending == 0 && endOp == ZSTD_e_end) c->emittedAny = false;        // the stream is complete: the next one starts fresh
    return pending;
}
size_t ZSTD_compressStream2(ZSTD_CCtx* c, ZSTD_outBuffer* out, ZSTD_inBuffer* in, ZSTD_EndDirective endOp) {
    try { return compress_stream2(c, out, in, endOp); } catch (...) { return ERR(E_memory_allocation); }
}
size_t ZSTD_compressStream(ZSTD_CStream* z, ZSTD_outBuffer* out, ZSTD_inBuffer* in) { return ZSTD_compressStream2(z, out, in, ZSTD_e_continue); }
size_t ZSTD_flushStream(ZSTD_CStream* z, ZSTD_outBuffer* out) { ZSTD_inBuffer in = { nullptr, 0, 0 }; return ZSTD_compressStream2(z, out, &in, ZSTD_e_flush); }
size_t ZSTD_endStream(ZSTD_CStream* z, ZSTD_outBuffer* out) { ZSTD_inBuffer in = { nullptr, 0, 0 }; return ZSTD_compressStream2(z, out, &in, ZSTD_e_end); }

ZSTD_DStream* ZSTD_createDStream(void) { return ZSTD_createDCtx(); }
size_t ZSTD_freeDStream(ZSTD_DStream* z) { return ZSTD_freeDCtx(z); }
size_t ZSTD_initDStream(ZSTD_DStream* z) { if (!z) return ERR(E_GENERIC); ZSTD_DCtx_reset(z, ZSTD_reset_session_only); return 5; }

// Decoding side.  Whole frames are decoded, as many as the offered input holds and one batch takes; only a frame cut by the end
// of the input is copied aside until the rest arrives.  Memory is bounded by what the blocks PRESENT in the input can regenerate
// (blocks x blockSizeMax): a frame header promising more than that is corruption, it never sizes an allocation.
// A frame of more blocks than one segment (zstdb200_fstream_blocks) goes to a frame stream instead, whether it is present whole or cut
// by the end of the input: its segments are decoded as their blocks arrive and handed out one after the other, in memory bounded by
// its window and one segment.
static size_t dstream_frame_bound(const FrameHeader& fh, size_t blocks, u64* bound) {
    if (fh.skippable) { *bound = 0; return 0; }
    u64 const byBlocks = (u64)blocks * fh.blockSizeMax;
    if (fh.hasContentSize && fh.contentSize > byBlocks) return ERR(E_corruption_detected);
    *bound = fh.hasContentSize ? fh.contentSize : byBlocks;
    return 0;
}
static size_t decompress_stream(ZSTD_DStream* d, ZSTD_outBuffer* out, ZSTD_inBuffer* in) {
    if (!d || !out || !in) return ERR(E_GENERIC);
    if (out->pos > out->size) return ERR(E_dstSize_tooSmall);
    if (in->pos > in->size) return ERR(E_srcSize_wrong);
    size_t const minHdr = d->format ? 1 : 5;          // ZSTD_startingInputLength
    size_t const maxPending = (size_t)1 << 31;        // compressed bytes of ONE frame this layer is willing to collect
    for (;;) {
        // drain regenerated bytes
        {   size_t const avail = d->outBuf.size() - d->outPos, room = out->size - out->pos;
            size_t const k = avail < room ? avail : room;
            if (k) { memcpy((u8*)out->dst + out->pos, d->outBuf.data() + d->outPos, k); out->pos += k; d->outPos += k; }
            if (d->outPos < d->outBuf.size()) return 1;   // more to flush
            d->outBuf.clear(); d->outPos = 0; }
        // a frame stream in progress takes the bytes put aside, then the caller's
        if (d->fs) {
            PooledCtx g(d->format ? FRAME_MAGICLESS : 0u, CParams{});
            if (!g.ok) return ERR(E_GENERIC);
            size_t r = 1;
            if (!d->inBuf.empty()) {
                size_t ip = 0;
                r = zstdb200_fstream_decode(g.c, d->fs, d->inBuf.data(), d->inBuf.size(), &ip, out->dst, out->size, &out->pos);
                d->inBuf.erase_front(ip);
            }
            if (r == 1 && d->inBuf.empty()) r = zstdb200_fstream_decode(g.c, d->fs, in->src, in->size, &in->pos, out->dst, out->size, &out->pos);
            if (r == 1) return 1;
            d->end_frame_stream();
            if (isErr(r)) return r;
            if (d->inBuf.empty() && in->pos == in->size) return 0;
            continue;                            // the frame is done: the bytes after it
        }
        // where the next frames are: the bytes put aside, or the caller's buffer
        bool const aside = !d->inBuf.empty();
        if (aside && in->pos < in->size) {       // complete the frame that was cut: take what its header / blocks say is missing
            size_t need = 1;
            if (d->inBuf.size() < minHdr) need = minHdr - d->inBuf.size();
            else {
                FrameHeader fh; size_t blocks = 0;
                size_t const fs = host_find_frame_size(d->inBuf.data(), d->inBuf.size(), &blocks, &fh, (u32)d->format, &need);
                if (!isErr(fs)) need = 0;
                else if (fs != ERR(E_srcSize_wrong)) return fs;      // otherwise `need` = bytes up to the next point where the walk can go on, never past the frame
            }
            if (need) {
                size_t k = in->size - in->pos; if (k > need) k = need;
                if (d->inBuf.size() + k > maxPending) return ERR(E_memory_allocation);
                d->inBuf.append((const u8*)in->src + in->pos, k);
                in->pos += k;
            }
        }
        const u8* const base = aside ? d->inBuf.data() : (const u8*)in->src + in->pos;
        size_t const have = aside ? d->inBuf.size() : in->size - in->pos;
        // a frame of more blocks than one segment, present whole or cut, that is the first here: it becomes the frame stream
        auto streams = [&](const FrameHeader& fh, size_t blocks) {
            if (blocks <= 1 || fh.skippable || fh.windowSize > d->maxWindowSize) return false;      // (fh is set once blocks are)
            if (!d->segBlocks) { PooledCtx g(0u, CParams{}); if (!g.ok) return false; d->segBlocks = zstdb200_fstream_blocks(g.c); }
            return blocks > d->segBlocks;
        };
        bool stream = false;
        // walk the whole frames present
        std::vector<size_t> fsz, cap, slot;
        size_t used = 0; u64 outTotal = 0;
        while (used < have && outTotal < stream_batch_bytes() && fsz.size() < 65536) {
            if (have - used < minHdr) break;
            FrameHeader fh; size_t blocks = 0;
            size_t const fs = host_find_frame_size(base + used, have - used, &blocks, &fh, (u32)d->format);
            if ((!isErr(fs) || fs == ERR(E_srcSize_wrong)) && streams(fh, blocks)) { stream = fsz.empty(); break; }
            if (isErr(fs)) { if (fs == ERR(E_srcSize_wrong)) break; if (fsz.empty()) return fs; break; }      // a later frame's error surfaces when it is first
            u64 bound = 0;
            {   size_t const r = dstream_frame_bound(fh, blocks, &bound); if (isErr(r)) { if (fsz.empty()) return r; break; } }
            // the reference refuses windows beyond ZSTD_d_windowLogMax unless the frame fits the caller's buffer in one pass (:2190-2228)
            if (!fh.skippable && fh.windowSize > d->maxWindowSize && !(fh.hasContentSize && (u64)(out->size - out->pos) >= fh.contentSize)) {
                if (fsz.empty()) return ERR(E_frameParameter_windowTooLarge);
                break;
            }
            fsz.push_back(fs); cap.push_back((size_t)bound); slot.push_back((size_t)bound); used += fs; outTotal += bound;
        }
        if (stream) {
            PooledCtx g(d->format ? FRAME_MAGICLESS : 0u, CParams{});
            if (!g.ok) return ERR(E_GENERIC);
            size_t const h = zstdb200_fstream_open(g.c, base, have, d->format, d->maxWindowSize, &d->fs);
            if (isErr(h)) return h;
            if (aside) d->inBuf.erase_front(h); else in->pos += h;
            continue;
        }
        if (!fsz.empty()) {
            // straight into the caller's buffer when everything fits there, else through outBuf
            bool const direct = out->size - out->pos >= outTotal;
            u8* const dstp = direct ? (u8*)out->dst + out->pos : (d->outBuf.resize((size_t)outTotal + 1), d->outBuf.data());
            PooledCtx g(d->format ? FRAME_MAGICLESS : 0u, CParams{});
            if (!g.ok) { d->outBuf.clear(); return ERR(E_GENERIC); }
            size_t const r = zstdb200_decompress_frames(g.c, base, fsz.data(), fsz.size(), dstp, (size_t)outTotal, cap.data());
            if (isErr(r)) { d->outBuf.clear(); return r; }
            // frames without a content size may regenerate less than their slot: close the gaps (cap[] holds the regenerated sizes now)
            size_t w = 0, rd = 0;
            for (size_t i = 0; i < fsz.size(); i++) {
                if (w != rd && cap[i]) memmove(dstp + w, dstp + rd, cap[i]);
                w += cap[i]; rd += slot[i];
            }
            if (direct) out->pos += w; else { d->outBuf.resize(w); d->outPos = 0; }
            if (aside) d->inBuf.erase_front(used);      // at most one frame was aside: this empties it or leaves a short tail
            else in->pos += used;
            if (d->outBuf.empty() && d->inBuf.empty() && in->pos == in->size) return 0;
            continue;
        }
        // no whole frame here
        if (aside) {
            if (in->pos == in->size) return d->inBuf.size() < minHdr ? minHdr - d->inBuf.size() : 1;
            continue;                            // more input was offered: keep completing the frame
        }
        if (have == 0) return 0;
        // the caller's buffer ends inside a frame: put that piece aside
        if (have > maxPending) return ERR(E_memory_allocation);
        d->inBuf.assign(base, have);
        in->pos += have;
        return d->inBuf.size() < minHdr ? minHdr - d->inBuf.size() : 1;
    }
}
size_t ZSTD_decompressStream(ZSTD_DStream* d, ZSTD_outBuffer* out, ZSTD_inBuffer* in) {
    try { return decompress_stream(d, out, in); } catch (...) { return ERR(E_memory_allocation); }
}

}  // extern "C"
