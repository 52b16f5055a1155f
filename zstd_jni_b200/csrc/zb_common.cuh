// zb_common.cuh -- shared definitions for the GPU Zstandard block codec.
//
// The codec is written as warp-cooperative __host__ __device__ templates over a
// "warp context" (lane id, lane count W, sync, broadcast).  On the GPU W = 32 and
// one warp owns one zstd frame; the host instantiation (W = 1, tests only, see
// tests/hostsim/) runs the very same source so that format logic can be checked
// on a machine without a GPU.  Product builds only ever launch the CUDA kernels.
//
// Reference behaviour being reproduced (N/ = luben/zstd-jni src/main/native/):
// constants N/common/zstd_internal.h:90-164, error codes N/zstd_errors.h:42-78.
#pragma once
#include <stddef.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define ZB_HD __host__ __device__ __forceinline__
#define ZB_HDN static __host__ __device__ __noinline__
#else
#define ZB_HD inline
#define ZB_HDN static
#endif

namespace zb {

typedef uint8_t u8;
typedef uint16_t u16;
typedef uint32_t u32;
typedef uint64_t u64;
typedef int64_t i64;
typedef int16_t i16;

// ---- error convention: (size_t)-code, N/common/error_private.h:49-54
enum : int {
    E_GENERIC = 1, E_prefix_unknown = 10, E_frameParameter_unsupported = 14, E_frameParameter_windowTooLarge = 16,
    E_corruption_detected = 20, E_checksum_wrong = 22, E_literals_headerWrong = 24, E_dictionary_corrupted = 30, E_dictionary_wrong = 32,
    E_parameter_unsupported = 40, E_parameter_outOfBound = 42, E_tableLog_tooLarge = 44, E_maxSymbolValue_tooLarge = 46,
    E_maxSymbolValue_tooSmall = 48, E_stage_wrong = 60, E_init_missing = 62, E_memory_allocation = 64, E_workSpace_tooSmall = 66,
    E_dstSize_tooSmall = 70, E_srcSize_wrong = 72, E_dstBuffer_null = 74, E_sequenceProducer_failed = 106, E_externalSequences_invalid = 107,
    E_maxCode = 120
};
ZB_HD size_t ERR(int code) { return (size_t)0 - (size_t)code; }
ZB_HD bool isErr(size_t c) { return c > ERR(E_maxCode); }

// ---- format constants
constexpr u32 BLOCKSIZE_MAX = 1u << 17;
constexpr u32 MINMATCH = 3;
constexpr u32 MaxLL = 35, MaxML = 52, MaxOff = 31, DefaultMaxOff = 28;
constexpr u32 LLFSELog = 9, MLFSELog = 9, OffFSELog = 8, LitHufLog = 11;
constexpr u32 LONGNBSEQ = 0x7F00;
constexpr u32 HUF_TABLELOG_MAX = 12;
constexpr u32 MAGIC = 0xFD2FB528u;

// ---- small intrinsics with host fallbacks
ZB_HD u32 highbit32(u32 v) {
#if defined(__CUDA_ARCH__)
    return 31u - (u32)__clz((int)v);
#else
    return 31u - (u32)__builtin_clz(v);
#endif
}
ZB_HD u32 ctz64(u64 v) {
#if defined(__CUDA_ARCH__)
    return (u32)__ffsll((long long)v) - 1u;
#else
    return (u32)__builtin_ctzll(v);
#endif
}
ZB_HD u32 popc32(u32 v) {
#if defined(__CUDA_ARCH__)
    return (u32)__popc(v);
#else
    return (u32)__builtin_popcount(v);
#endif
}
ZB_HD u32 ctz32(u32 v) {   // v != 0
#if defined(__CUDA_ARCH__)
    return (u32)__ffs((int)v) - 1u;
#else
    return (u32)__builtin_ctz(v);
#endif
}
ZB_HD u32 umin(u32 a, u32 b) { return a < b ? a : b; }
ZB_HD u32 umax(u32 a, u32 b) { return a > b ? a : b; }

// Unaligned little-endian loads built from aligned 8-byte words: the GPU faults on
// misaligned wide loads, and an aligned word that holds at least one valid byte is
// always inside the same allocation (cudaMalloc / caching allocators round to >=256 B).
ZB_HD u64 ld_aligned64(const u8* p) { return *reinterpret_cast<const u64*>(p); }
// Random single-word probes (hash-table cells): cache in L2 only.  Through L1 every miss pulls a whole 128-byte
// line over the crossbar and out of HBM for 4 useful bytes (measured: 3x the requested sectors, profiles/).
ZB_HD void prefetch_l2(const void* p) {
#if defined(__CUDA_ARCH__)
    asm volatile("prefetch.global.L2 [%0];" :: "l"(p));
#else
    (void)p;
#endif
}
ZB_HD u32 ld_probe32(const u32* p) {
#if defined(__CUDA_ARCH__) && defined(ZB_TABLES_MAY_BE_SHARED)
    return __isShared(p) ? *p : __ldcg(p);          // (experiment: level-1 table in shared memory, k_parse_fast_smem)
#elif defined(__CUDA_ARCH__)
    return __ldcg(p);
#else
    return *p;
#endif
}
// Device: from aligned 4-byte words and funnel shifts (three loads and two shifts for eight bytes; the 64-bit form costs two 8-byte
// loads plus four shifts and the 64-bit arithmetic around them); a word is only touched when it holds a wanted byte.
ZB_HD u64 load64(const u8* p) {
    uintptr_t const a = reinterpret_cast<uintptr_t>(p);
#if defined(__CUDA_ARCH__)
    const u32* const w = reinterpret_cast<const u32*>(a & ~(uintptr_t)3);
    u32 const sh = (u32)(a & 3) * 8;
    u32 const w0 = w[0], w1 = w[1], w2 = sh ? w[2] : 0u;
    return (u64)__funnelshift_r(w0, w1, sh) | ((u64)__funnelshift_r(w1, w2, sh) << 32);
#else
    u32 const sh = (u32)(a & 7) * 8;
    const u8* const A = reinterpret_cast<const u8*>(a & ~(uintptr_t)7);
    u64 const lo = ld_aligned64(A);
    if (sh == 0) return lo;
    return (lo >> sh) | (ld_aligned64(A + 8) << (64 - sh));
#endif
}
// Same, but never touches a word beyond the first `nbytes` (1..8) bytes.
ZB_HD u64 load64_n(const u8* p, u32 nbytes) {
    uintptr_t const a = reinterpret_cast<uintptr_t>(p);
#if defined(__CUDA_ARCH__)
    const u32* const w = reinterpret_cast<const u32*>(a & ~(uintptr_t)3);
    u32 const o = (u32)(a & 3), sh = o * 8;
    u32 const w0 = w[0], w1 = o + nbytes > 4 ? w[1] : 0u, w2 = o + nbytes > 8 ? w[2] : 0u;
    return (u64)__funnelshift_r(w0, w1, sh) | ((u64)__funnelshift_r(w1, w2, sh) << 32);
#else
    u32 const o = (u32)(a & 7);
    const u8* const A = reinterpret_cast<const u8*>(a & ~(uintptr_t)7);
    u64 v = ld_aligned64(A) >> (o * 8);
    if (o + nbytes > 8) v |= ld_aligned64(A + 8) << (64 - o * 8);
    return v;
#endif
}
ZB_HD u32 load32(const u8* p) {
#if defined(__CUDA_ARCH__)
    uintptr_t const a = reinterpret_cast<uintptr_t>(p);
    const u32* const w = reinterpret_cast<const u32*>(a & ~(uintptr_t)3);
    u32 const sh = (u32)(a & 3) * 8;
    return __funnelshift_r(w[0], sh ? w[1] : 0u, sh);
#else
    return (u32)load64_n(p, 4);
#endif
}
ZB_HD u32 load24(const u8* p) { return (u32)load64_n(p, 3) & 0xFFFFFFu; }
ZB_HD u32 load16(const u8* p) { return (u32)load64_n(p, 2) & 0xFFFFu; }

// bits [lo, lo+n) of the little-endian bit array at p; n <= 57; lo may be negative
// (bits below 0 read as zero, mirroring the reference's zero-filled container once
// a backward stream is exhausted, N/common/bitstream.h:344-351).
ZB_HD u64 peek_bits(const u8* p, i64 lo, u32 n) {
    if (n == 0) return 0;
    if (lo < 0) {
        i64 const miss = -lo;
        if (miss >= (i64)n) return 0;
        return peek_bits(p, 0, n - (u32)miss) << miss;
    }
    const u8* const q = p + (lo >> 3);
    u32 const sh = (u32)(lo & 7);
    u64 const w = load64_n(q, (sh + n + 7) >> 3);
    return (w >> sh) & ((n >= 64) ? ~0ull : ((1ull << n) - 1));
}

// ---------------------------------------------------------------- XXH64
// published xxHash64 (N/common/xxhash.h), serial; only used when the frame asks for it.
ZB_HD u64 rotl64(u64 x, int r) { return (x << r) | (x >> (64 - r)); }
ZB_HDN u64 xxh64(const u8* p, size_t len) {
    constexpr u64 P1 = 0x9E3779B185EBCA87ULL, P2 = 0xC2B2AE3D27D4EB4FULL, P3 = 0x165667B19E3779F9ULL, P4 = 0x85EBCA77C2B2AE63ULL, P5 = 0x27D4EB2F165667C5ULL;
    const u8* const end = p + len; u64 h;
    auto rnd = [&](u64 acc, u64 in) { acc += in * P2; acc = rotl64(acc, 31); return acc * P1; };
    auto mrg = [&](u64 acc, u64 v) { v = rnd(0, v); acc ^= v; return acc * P1 + P4; };
    if (len >= 32) {
        u64 v1 = P1 + P2, v2 = P2, v3 = 0, v4 = 0 - P1;
        do { v1 = rnd(v1, load64(p)); v2 = rnd(v2, load64(p + 8)); v3 = rnd(v3, load64(p + 16)); v4 = rnd(v4, load64(p + 24)); p += 32; } while (p + 32 <= end);
        h = rotl64(v1, 1) + rotl64(v2, 7) + rotl64(v3, 12) + rotl64(v4, 18);
        h = mrg(h, v1); h = mrg(h, v2); h = mrg(h, v3); h = mrg(h, v4);
    } else h = P5;
    h += (u64)len;
    while (p + 8 <= end) { h ^= rnd(0, load64_n(p, 8)); h = rotl64(h, 27) * P1 + P4; p += 8; }
    if (p + 4 <= end) { h ^= (u64)load32(p) * P1; h = rotl64(h, 23) * P2 + P3; p += 4; }
    while (p < end) { h ^= (*p++) * P5; h = rotl64(h, 11) * P1; }
    h ^= h >> 33; h *= P2; h ^= h >> 29; h *= P3; h ^= h >> 32;
    return h;
}

// ---- backward bit reader of ONE thread, all in 32-bit registers.
// The serial chains of the format (Huffman symbol -> bit count -> next symbol; FSE state -> bit counts -> bits ->
// state) are latency chains: a memory load or a 64-bit shift sequence on them multiplies the cost of every symbol.
// Here the next bits always sit in the register pair hi:lo (c = bits of hi already consumed, 0..31); reading is one
// funnel shift, and the word that slides in next (nx) was loaded two words -- hundreds of cycles -- before it is
// needed, so no load is ever waited for.  Bits below the first byte of the stream read as zero and `pos` keeps
// counting down, mirroring the reference's zero-filled container (N/common/bitstream.h:344-351).
ZB_HD u32 fshl32(u32 lo, u32 hi, u32 s) {      // upper 32 bits of (hi:lo) << s, s in 0..31
#if defined(__CUDA_ARCH__)
    return __funnelshift_l(lo, hi, s);
#else
    return s ? (hi << s) | (lo >> (32 - s)) : hi;
#endif
}
ZB_HD u32 fshr32(u32 lo, u32 hi, u32 s) {      // lower 32 bits of (hi:lo) >> s, s in 0..31
#if defined(__CUDA_ARCH__)
    return __funnelshift_r(lo, hi, s);
#else
    return s ? (lo >> s) | (hi << (32 - s)) : lo;
#endif
}
// Forward copy of n bytes from m to t by ONE thread with the semantics of a byte-by-byte loop (so an overlapping
// source, t - m < n, replicates its period like ZSTD_execSequence's match copy), but moving aligned 32-bit words
// whenever the distance allows it: head bytes until t is word aligned, then one aligned store per word fed by two
// aligned loads and a funnel shift, then the tail.  The aligned loads may touch up to 3 bytes on either side of
// the source range inside words that also hold requested bytes; callers guarantee those words are mapped.
ZB_HD void copy_fwd(u8* t, const u8* m, u32 n) {
    uintptr_t const off = (uintptr_t)(t - m);
    if (off < 8 && n > off) { for (u32 k = 0; k < n; k++) t[k] = m[k]; return; }     // short period: replicate byte by byte
    u32 k = 0;
    if (n > 16) {      // long: aligned words
        while ((reinterpret_cast<uintptr_t>(t + k) & 3) != 0) { t[k] = m[k]; k++; }
        u32 const sh = (u32)(reinterpret_cast<uintptr_t>(m + k) & 3) * 8;
        const u8* a = m + k - (sh >> 3);
        for (; k + 4 <= n; k += 4, a += 4) {
            u32 const w0 = *reinterpret_cast<const u32*>(a);
            u32 const w1 = sh ? *reinterpret_cast<const u32*>(a + 4) : 0;
            *reinterpret_cast<u32*>(t + k) = fshr32(w0, w1, sh);
        }
    }
    // short (and the tail of long): eight source bytes per step come from one unaligned read, the stores are
    // independent of each other, so there is no load -> store -> load chain
    for (; k < n; k += 8) {
        u32 const r = n - k < 8 ? n - k : 8;
        u64 const v = load64_n(m + k, r);
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
        for (u32 j = 0; j < 8; j++) if (j < r) t[k + j] = (u8)(v >> (8 * j));
    }
}

struct BackBits {
    const u32* W; int wp; u32 firstMask;
    u32 hi, lo, nx, nmask, c;         // nx is kept as loaded; its mask is applied one step later, when it moves into lo,
                                      // so that nothing consumes a load result in the step that issued the load
    int pos;                          // stream bits not yet consumed (negative once the stream is overrun)
    ZB_HD u32 raw(int k) const { u32 v = 0; if (k >= 0) v = W[k]; return v; }
    ZB_HD u32 mask_of(int k) const { return k == 0 ? firstMask : 0xFFFFFFFFu; }
    ZB_HD void init(const u8* ip, int bits) {
        uintptr_t const a = reinterpret_cast<uintptr_t>(ip);
        W = reinterpret_cast<const u32*>(a & ~(uintptr_t)3);
        u32 const sb = (u32)(a & 3);
        firstMask = 0xFFFFFFFFu << (8 * sb);
        pos = bits;
        int const gpos = bits + 8 * (int)sb;
        if (gpos <= 0) { hi = lo = nx = 0; nmask = 0; c = 0; wp = -1; return; }
        int const k0 = (gpos - 1) >> 5;
        c = 32u - (u32)(gpos - 32 * k0);          // bits of the top word above the end mark count as consumed
        hi = raw(k0) & mask_of(k0); lo = raw(k0 - 1) & mask_of(k0 - 1); nx = raw(k0 - 2); nmask = mask_of(k0 - 2); wp = k0 - 2;
#if defined(__CUDA_ARCH__)
        for (int k = k0 - 32; k >= 0 && k >= k0 - 96; k -= 32) asm volatile("prefetch.L1 [%0];" :: "l"(W + k));
#endif
    }
    ZB_HD u32 peek32() const { return fshl32(lo, hi, c); }      // the next 32 bits, first bit on top
    ZB_HD void skip(u32 n) {                                    // n <= 32
        c += n; pos -= (int)n;
        if (c >= 32) {
            c -= 32; hi = lo; lo = nx & nmask; wp--; nx = raw(wp); nmask = mask_of(wp);
#if defined(__CUDA_ARCH__)
            // The lanes of a warp read 32 different streams and step in lockstep: one lane's cache miss stalls all of
            // them, so every 64 bytes the line two ahead (256 B below) is pulled into L1 long before it is needed.
            if ((wp & 15) == 0 && wp >= 64) asm volatile("prefetch.L1 [%0];" :: "l"(W + (wp - 64)));
#endif
        }
    }
    ZB_HD u32 take(u32 n) {                                     // n in 0..32
        u32 const w32 = peek32();
        u32 const v = n ? w32 >> (32 - n) : 0;
        skip(n);
        return v;
    }
};

// ---- per-code extra bits / base values (N/common/zstd_internal.h:119-144; OF: code == bits)
struct CodeTables {
    u8 LL_bits[MaxLL + 1];
    u8 ML_bits[MaxML + 1];
    u32 LL_base[MaxLL + 1];
    u32 ML_base[MaxML + 1];
    i16 LL_defaultNorm[MaxLL + 1];
    i16 ML_defaultNorm[MaxML + 1];
    i16 OF_defaultNorm[DefaultMaxOff + 1];
};

// One initializer shared by the __constant__ copy (device) and the host copy.
#define ZB_CODE_TABLES_INIT { \
    {0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,1,1,1,1,2,2,3,3,4,6,7,8,9,10,11,12,13,14,15,16}, \
    {0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,1,1,1,1,2,2,3,3,4,4,5,7,8,9,10,11,12,13,14,15,16}, \
    {0,1,2,3,4,5,6,7,8,9,10,11,12,13,14,15,16,18,20,22,24,28,32,40,48,64,128,256,512,1024,2048,4096,8192,16384,32768,65536}, \
    {3,4,5,6,7,8,9,10,11,12,13,14,15,16,17,18,19,20,21,22,23,24,25,26,27,28,29,30,31,32,33,34,35,37,39,41,43,47,51,59,67,83,99,131,259,515,1027,2051,4099,8195,16387,32771,65539}, \
    {4,3,2,2,2,2,2,2,2,2,2,2,2,1,1,1,2,2,2,2,2,2,2,2,2,3,2,1,1,1,1,1,-1,-1,-1,-1}, \
    {1,4,3,2,2,2,2,2,2,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,-1,-1,-1,-1,-1,-1,-1}, \
    {1,1,1,1,1,1,2,2,2,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,-1,-1,-1,-1,-1} }
#if defined(__CUDACC__)
static __constant__ CodeTables c_tables = ZB_CODE_TABLES_INIT;
#endif
static const CodeTables h_tables = ZB_CODE_TABLES_INIT;
#if defined(__CUDA_ARCH__)
#define ZB_T (::zb::c_tables)
#else
#define ZB_T (::zb::h_tables)
#endif

// floor(-log2(x / 256) * 256) for x in [0, 256), 0 for x == 0 (kInverseProbabilityLog256, N/compress/zstd_compress_sequences.c:21-44)
struct InvProbTable { u16 v[256]; };
#define ZB_INVPROB_INIT { { \
    0,    2048, 1792, 1642, 1536, 1453, 1386, 1329, 1280, 1236, 1197, 1162, 1130, 1100, 1073, 1047, 1024, 1001, 980,  960,  941,  923,  906,  889, \
    874,  859,  844,  830,  817,  804,  791,  779,  768,  756,  745,  734,  724,  714,  704,  694,  685,  676,  667,  658,  650,  642,  633,  626, \
    618,  610,  603,  595,  588,  581,  574,  567,  561,  554,  548,  542,  535,  529,  523,  517,  512,  506,  500,  495,  489,  484,  478,  473, \
    468,  463,  458,  453,  448,  443,  438,  434,  429,  424,  420,  415,  411,  407,  402,  398,  394,  390,  386,  382,  377,  373,  370,  366, \
    362,  358,  354,  350,  347,  343,  339,  336,  332,  329,  325,  322,  318,  315,  311,  308,  305,  302,  298,  295,  292,  289,  286,  282, \
    279,  276,  273,  270,  267,  264,  261,  258,  256,  253,  250,  247,  244,  241,  239,  236,  233,  230,  228,  225,  222,  220,  217,  215, \
    212,  209,  207,  204,  202,  199,  197,  194,  192,  190,  187,  185,  182,  180,  178,  175,  173,  171,  168,  166,  164,  162,  159,  157, \
    155,  153,  151,  149,  146,  144,  142,  140,  138,  136,  134,  132,  130,  128,  126,  123,  121,  119,  117,  115,  114,  112,  110,  108, \
    106,  104,  102,  100,  98,   96,   94,   93,   91,   89,   87,   85,   83,   82,   80,   78,   76,   74,   73,   71,   69,   67,   66,   64, \
    62,   61,   59,   57,   55,   54,   52,   50,   49,   47,   46,   44,   42,   41,   39,   37,   36,   34,   33,   31,   30,   28,   26,   25, \
    23,   22,   20,   19,   17,   16,   14,   13,   11,   10,   8,    7,    5,    4,    2,    1 } }
#if defined(__CUDACC__)
static __constant__ InvProbTable c_invprob = ZB_INVPROB_INIT;
#endif
static const InvProbTable h_invprob = ZB_INVPROB_INIT;
#if defined(__CUDA_ARCH__)
#define ZB_INVPROB (::zb::c_invprob.v)
#else
#define ZB_INVPROB (::zb::h_invprob.v)
#endif

// ---- optional per-phase cycle counters (profiling builds only: -DZB_PHASE_TIMERS; scripts/gpu_phases.sh)
#if defined(ZB_PHASE_TIMERS) && defined(__CUDACC__)
__device__ unsigned long long g_phaseCycles[16];
#endif
#if defined(ZB_PHASE_TIMERS) && defined(__CUDA_ARCH__)
#define ZB_PT_DECL long long zb_pt0 = clock64();
#define ZB_PT(k) do { long long const zb_t = clock64(); if ((threadIdx.x & 31) == 0) atomicAdd(&::zb::g_phaseCycles[k], (unsigned long long)(zb_t - zb_pt0)); zb_pt0 = zb_t; } while (0)
#else
#define ZB_PT_DECL
#define ZB_PT(k) do {} while (0)
#endif

// ---- warp contexts
#if defined(__CUDACC__)
// LANES consecutive lanes of a hardware warp acting as one cooperative group (LANES = 32: the whole warp).
// Collectives name only the group's lanes, so several groups of one warp may diverge freely (sm_70+).
template <int LANES>
struct GroupDev {
    int lane;        // lane inside the group
    u32 gmask;       // the group's lanes inside the hardware warp
    int gshift;      // first lane of the group
    static constexpr int W = LANES;
    static constexpr u32 FULL = (LANES >= 32) ? 0xFFFFFFFFu : ((1u << (LANES & 31)) - 1);
    __device__ __forceinline__ static GroupDev make() {
        int const l = (int)(threadIdx.x & 31), sh = l & ~(LANES - 1);
        return GroupDev{l & (LANES - 1), (LANES >= 32) ? 0xFFFFFFFFu : (FULL << sh), sh};
    }
    // A whole-warp group has a constant mask and shift.  Kernels pass the group by reference into non-inlined parsers, where
    // the fields live on the stack and are reloaded after every global store, in front of the next collective.
    __device__ __forceinline__ u32 mask() const { return LANES >= 32 ? 0xFFFFFFFFu : gmask; }
    __device__ __forceinline__ int shift() const { return LANES >= 32 ? 0 : gshift; }
    __device__ __forceinline__ void sync() const { __syncwarp(mask()); }
    template <class T> __device__ __forceinline__ T shfl(T v, int src) const { return __shfl_sync(mask(), v, src, LANES); }
    template <class T> __device__ __forceinline__ T bcast(T v, int src = 0) const { return __shfl_sync(mask(), v, src, LANES); }
    __device__ __forceinline__ u32 ballot(bool p) const { return (__ballot_sync(mask(), p) >> shift()) & FULL; }
    __device__ __forceinline__ u32 match_any(u32 v) const { return (__match_any_sync(mask(), v) >> shift()) & FULL; }
    __device__ __forceinline__ u32 sum(u32 v) const {
        for (int o = LANES / 2; o > 0; o >>= 1) v += __shfl_xor_sync(mask(), v, o, LANES);
        return v;
    }
    __device__ __forceinline__ u32 max(u32 v) const {
        for (int o = LANES / 2; o > 0; o >>= 1) { u32 t = __shfl_xor_sync(mask(), v, o, LANES); v = t > v ? t : v; }
        return v;
    }
    __device__ __forceinline__ void atomic_inc(u32* p) const { atomicAdd(p, 1u); }
    __device__ __forceinline__ void atomic_add(u32* p, u32 v) const { atomicAdd(p, v); }
    // exclusive prefix sum over the group's lanes
    __device__ __forceinline__ u32 exscan(u32 v) const {
        u32 x = v;
        for (int o = 1; o < LANES; o <<= 1) { u32 const t = __shfl_up_sync(mask(), x, o, LANES); if (lane >= o) x += t; }
        return x - v;
    }
    // OR one byte into memory shared with neighbouring lanes (32-bit atomic on the containing word)
    __device__ __forceinline__ void atomic_or32(u32* p, u32 v) const { atomicOr(p, v); }
    __device__ __forceinline__ void atomic_or_byte(u8* p, u32 v) const {
        uintptr_t const a = reinterpret_cast<uintptr_t>(p);
        atomicOr(reinterpret_cast<unsigned int*>(a & ~(uintptr_t)3), v << (8 * (u32)(a & 3)));
    }
};
typedef GroupDev<32> WarpDev;
#endif
// The calling lane's index in its group.  A device group derives it from the thread index instead of reading the field, which
// lives on the stack in non-inlined parsers (and waits there behind every global store).
template <class C> ZB_HD u32 lane_of(const C& w) { return (u32)w.lane; }
#if defined(__CUDACC__)
template <int LANES> __device__ __forceinline__ u32 lane_of(const GroupDev<LANES>&) { return threadIdx.x & (u32)(LANES - 1); }
#endif
struct WarpHost {
    int lane = 0;
    static constexpr int W = 1;
    static constexpr u32 FULL = 1u;
    void sync() const {}
    template <class T> T bcast(T v, int = 0) const { return v; }
    template <class T> T shfl(T v, int) const { return v; }
    u32 match_any(u32) const { return 1u; }
    u32 ballot(bool p) const { return p ? 1u : 0u; }
    u32 sum(u32 v) const { return v; }
    u32 max(u32 v) const { return v; }
    void atomic_inc(u32* p) const { ++*p; }
    void atomic_add(u32* p, u32 v) const { *p += v; }
    u32 exscan(u32) const { return 0; }
    void atomic_or32(u32* p, u32 v) const { *p |= v; }
    void atomic_or_byte(u8* p, u32 v) const { *p = (u8)(*p | v); }
};

// Cooperative copy of n bytes between regions that do not overlap, any alignment on either side: head bytes until dst sits on a
// 16-byte boundary, then 16 bytes per lane and step (two unaligned 8-byte reads, two aligned 8-byte stores), then the tail.  The
// aligned reads may touch up to 7 bytes past the source range inside words that also hold requested bytes (see load64).
template <class C>
ZB_HD void wcopy(const C& w, u8* dst, const u8* src, size_t n) {
    size_t head = (size_t)((16 - (reinterpret_cast<uintptr_t>(dst) & 15)) & 15); if (head > n) head = n;
    for (size_t i = (size_t)w.lane; i < head; i += C::W) dst[i] = src[i];
    size_t const body = (n - head) / 16;
    u64* const d8 = reinterpret_cast<u64*>(dst + head); const u8* const s = src + head;
    for (size_t j = (size_t)w.lane; j < body; j += C::W) { u64 const lo = load64(s + 16 * j), hi = load64(s + 16 * j + 8); d8[2 * j] = lo; d8[2 * j + 1] = hi; }
    for (size_t i = head + body * 16 + (size_t)w.lane; i < n; i += C::W) dst[i] = src[i];
}

}  // namespace zb
