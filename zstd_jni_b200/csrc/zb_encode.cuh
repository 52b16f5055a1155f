// zb_encode.cuh -- warp-cooperative one-shot Zstandard frame encoder for inputs of at
// most one block (<= 128 KB): the unit of work of the batch API.  The emitted frame is
// byte-identical to the reference's ZSTD_compress2(chunk, level) for the negative levels and
// levels 1..12 (1..10 on inputs <= 16 KB), i.e. every strategy below the optimal parser.
//
// Reference decisions being reproduced (N/ = luben/zstd-jni src/main/native/):
//   parameters     N/compress/clevels.h:78-130, N/compress/zstd_compress.c:1472-1609,7759-7782
//   framing        N/compress/zstd_compress.c:4591-4743,5344-5381
//   parsers        N/compress/zstd_double_fast.c:105-323 (dfast), N/compress/zstd_fast.c:190-423 (fast),
//                  N/compress/zstd_lazy.c:1516-1779 (greedy/lazy/lazy2/btlazy2) with the row-based (:775-1283),
//                  hash-chain (:620-733) and binary-tree (:22-408) match finders
//   literals       N/compress/zstd_compress_literals.c:129-235, N/compress/huf_compress.c:146-1434, N/compress/hist.c
//   sequences      N/compress/zstd_compress.c:2693-3042, N/compress/zstd_compress_sequences.c:17-382,
//                  N/compress/fse_compress.c:68-525
//
// GPU mapping (W = 32 lanes, one warp per frame):
//   * dfast / fast: a batch of consecutive search positions is probed by consecutive lanes; pending table writes are
//     forwarded between lanes (__match_any_sync), the first event in the reference's order ends the batch and only
//     what the serial code would have written is committed (parse_dfast_warp, parse_fast_warp);
//   * lazy family with the row finder: sequential control flow executed uniformly, the row search spread over the
//     lanes (parse_lazy_warp); hash-chain and binary-tree finders run on lane 0;
//   * literal gathering, histograms, code computation, bit packing of the Huffman and sequence streams run on all
//     lanes (lane slices + exclusive-scan bit offsets); Huffman tree / FSE normalisation / table descriptions are
//     scalar jobs on lane 0 in shared memory; the three FSE state chains run on lanes 0..2;
//   * the serial variants (parse_dfast, parse_fast, parse_lazy) are the 1-lane host instantiation used by the tests.
#pragma once
#include "zb_common.cuh"

namespace zb {

struct CParams {
    u32 windowLog, chainLog, hashLog, searchLog, minMatch, targetLength, strategy;
    ZB_HD bool any_set() const { return (windowLog | chainLog | hashLog | searchLog | minMatch | targetLength | strategy) != 0; }      // as overrides (0 = from the level)
};
enum : u32 { S_fast = 1, S_dfast = 2, S_greedy = 3, S_lazy = 4, S_lazy2 = 5, S_btlazy2 = 6 };

// The explicit compression parameters in the order of ZSTD_c_windowLog (101) ... ZSTD_c_strategy (107): option name of
// zstdb200_set_option, field, and the bounds of ZSTD_cParam_getBounds (N/compress/zstd_compress.c:420-520); 0 is always accepted.
struct CParamBound { const char* option; u32 CParams::*member; int lo, hi;
                     bool accepts(long long v) const { return v == 0 || (v >= lo && v <= hi); } };
static const CParamBound CPARAM_BOUNDS[7] = {
    { "c_windowLog", &CParams::windowLog, 10, 31 }, { "c_hashLog", &CParams::hashLog, 6, 30 }, { "c_chainLog", &CParams::chainLog, 6, 30 },
    { "c_searchLog", &CParams::searchLog, 1, 30 }, { "c_minMatch", &CParams::minMatch, 3, 7 }, { "c_targetLength", &CParams::targetLength, 0, 131072 },
    { "c_strategy", &CParams::strategy, 1, 9 } };

constexpr u32 MAX_SEQ = (BLOCKSIZE_MAX / 4) + 8;
constexpr u32 PARSE_SKIPPED = 0xFFFFFFFFu;     // nbSeq marker: srcSize < 7, the block is stored raw (ZSTD_buildSeqStore :3273-3280)
constexpr u32 ENC_HASHLOG_MAX = 18;     // largest hashLog / chainLog of the supported rows

// ZSTD_getCParams_internal (:7759-7782) + ZSTD_adjustCParams_internal (:1472-1609) for a known
// srcSize <= 128 KB, no dictionary.  Returns false when the level selects a parser this build lacks.
// Level tables (clevels.h:78-92,104-116) in constant memory on the device, as a plain static on the host.
struct LevelTables { CParams t128[13]; CParams t16[11]; };
#define ZB_LEVEL_TABLES_INIT { { {17,12,12,1,5,1,S_fast}, {17,12,13,1,6,0,S_fast}, {17,13,15,1,5,0,S_fast}, {17,15,16,2,5,0,S_dfast}, {17,17,17,2,4,0,S_dfast}, \
                               {17,16,17,3,4,2,S_greedy}, {17,16,17,3,4,4,S_lazy}, {17,16,17,3,4,8,S_lazy2}, {17,16,17,4,4,8,S_lazy2}, {17,16,17,5,4,8,S_lazy2}, \
                               {17,16,17,6,4,8,S_lazy2}, {17,17,17,5,4,8,S_btlazy2}, {17,18,17,7,4,12,S_btlazy2} }, \
                               { {14,12,13,1,5,1,S_fast}, {14,14,15,1,5,0,S_fast}, {14,14,15,1,4,0,S_fast}, {14,14,15,2,4,0,S_dfast}, \
                             {14,14,14,4,4,2,S_greedy}, {14,14,14,3,4,4,S_lazy}, {14,14,14,4,4,8,S_lazy2}, {14,14,14,6,4,8,S_lazy2}, {14,14,14,8,4,8,S_lazy2}, \
                              {14,15,14,5,4,8,S_btlazy2}, {14,15,14,9,4,8,S_btlazy2} } }
#if defined(__CUDACC__)
static __constant__ LevelTables c_levels = ZB_LEVEL_TABLES_INIT;
#endif
static const LevelTables h_levels = ZB_LEVEL_TABLES_INIT;
#if defined(__CUDA_ARCH__)
#define ZB_LEVELS (::zb::c_levels)
#else
#define ZB_LEVELS (::zb::h_levels)
#endif

// ZSTD_adjustCParams_internal :1472-1609 for a known srcSize <= 128 KB without dictionary (the row-hash cap :1596-1606
// cannot bind: hashLog <= windowLog + 1 <= 18)
ZB_HD void adjust_cparams(CParams& cp, size_t srcSize) {
    u32 const tSize = (u32)srcSize;
    u32 const srcLog = (tSize < 64) ? 6 : highbit32(tSize - 1) + 1;
    if (cp.windowLog > srcLog) cp.windowLog = srcLog;
    if (cp.hashLog > cp.windowLog + 1) cp.hashLog = cp.windowLog + 1;
    {   u32 const cycleLog = cp.chainLog - (cp.strategy >= S_btlazy2 ? 1 : 0);      // ZSTD_cycleLog
        if (cycleLog > cp.windowLog) cp.chainLog -= (cycleLog - cp.windowLog); }
    if (cp.windowLog < 10) cp.windowLog = 10;
}

// `ov`: explicit parameters (ZSTD_c_windowLog ... ZSTD_c_strategy, 0 = not set) as ZSTD_getCParamsFromCCtxParams :1637-1651
// applies them: over the adjusted row of the level (ZSTD_overrideCParams :1623-1635), then adjusted again.
// checkWindow: refuse parameter sets whose window does not cover the input (matches would have to respect a sliding
// window inside the block, which these parsers do not implement).
ZB_HDN bool get_cparams(CParams* out, int level, size_t srcSize, const CParams* ov = nullptr, bool checkWindow = true) {
    // rows 0..12 of the "<=128 KB" table and 0..10 of the "<=16 KB" table (clevels.h:78-92,104-116).  greedy / lazy / lazy2
    // run with the row-based match finder when windowLog > 14 (ZSTD_resolveRowMatchFinderMode, zstd_compress.c:238-245),
    // i.e. for every srcSize > 16 KB, and with the hash-chain finder below; btlazy2 uses the binary tree.  The rows from
    // btopt on (optimal parser) are not built.
    if (srcSize > BLOCKSIZE_MAX) return false;
    int row = level;
    if (level == 0) row = 3;
    if (level < 0) row = 0;
    bool const small = srcSize <= 16 * 1024;
    if (row > (small ? 10 : 12)) return false;
    CParams cp = small ? ZB_LEVELS.t16[row] : ZB_LEVELS.t128[row];
    if (level < 0) { int const l = level < -(1 << 17) ? -(1 << 17) : level; cp.targetLength = (u32)(-l); }
    adjust_cparams(cp, srcSize);
    if (ov) {
        if (ov->windowLog) cp.windowLog = ov->windowLog;
        if (ov->hashLog) cp.hashLog = ov->hashLog;
        if (ov->chainLog) cp.chainLog = ov->chainLog;
        if (ov->searchLog) cp.searchLog = ov->searchLog;
        if (ov->minMatch) cp.minMatch = ov->minMatch;
        if (ov->targetLength) cp.targetLength = ov->targetLength;
        if (ov->strategy) cp.strategy = ov->strategy;
        if (cp.strategy > S_btlazy2) return false;
        adjust_cparams(cp, srcSize);
        if (checkWindow && ((size_t)1 << cp.windowLog) < srcSize) return false;
    }
    *out = cp;
    return true;
}

ZB_HD size_t compress_bound(size_t n) { return n + (n >> 8) + (n < (128u << 10) ? (((128u << 10) - n) >> 11) : 0); }

// ---- per-warp global workspace (carved by the host, see zb_capi.cu)
// One sequence as the parsers hand it to the entropy stage: 16 bytes, so that storing it is a single request (three
// 4-byte stores to three arrays were 14 % of the write requests of the parse kernel) and a row of sequences is read with
// one 16-byte load per lane.
struct alignas(16) Seq { u32 ll, of, ml, pad; };      // litLength, offBase, matchLength
struct EncWork {
    u32* hashLong;      // 1 << ENC_HASHLOG_MAX entries, zeroed by the kernel per frame (only the used part)
    u32* hashSmall;     // 1 << ENC_HASHLOG_MAX entries
    Seq* seq;           // MAX_SEQ records
    ZB_HD void put(u32 i, u32 ll, u32 of, u32 ml) const { Seq q; q.ll = ll; q.of = of; q.ml = ml; q.pad = 0; seq[i] = q; }
    ZB_HD Seq get(u32 i) const { return seq[i]; }
    u8* lit;            // BLOCKSIZE_MAX + 32
    u8* codes;          // 3 * MAX_SEQ
    u16* stbits;        // 3 * MAX_SEQ : per sequence and stream, FSE state bits (value | nbBits << 12)
};
ZB_HD size_t enc_entropy_work_bytes() { return (size_t)(BLOCKSIZE_MAX + 32) + 3 * (size_t)MAX_SEQ + 64 + 6 * (size_t)MAX_SEQ + 64; }
ZB_HD void enc_entropy_work_carve(EncWork& w, u8* base) {
    w.lit = base; base += BLOCKSIZE_MAX + 32;
    w.codes = base; base += 3 * (size_t)MAX_SEQ + 64;
    base = reinterpret_cast<u8*>((reinterpret_cast<uintptr_t>(base) + 15) & ~(uintptr_t)15);
    w.stbits = reinterpret_cast<u16*>(base);
}
ZB_HD size_t enc_work_bytes() {
    return (size_t)2 * (4u << ENC_HASHLOG_MAX) + (size_t)16 * MAX_SEQ + enc_entropy_work_bytes() + 64;
}
ZB_HD EncWork enc_work_carve(u8* base) {
    EncWork w;
    w.hashLong = reinterpret_cast<u32*>(base); base += (size_t)4 << ENC_HASHLOG_MAX;
    w.hashSmall = reinterpret_cast<u32*>(base); base += (size_t)4 << ENC_HASHLOG_MAX;
    w.seq = reinterpret_cast<Seq*>(base); base += 16 * (size_t)MAX_SEQ;
    enc_entropy_work_carve(w, base);
    return w;
}

// ---- per-warp shared scratch
struct HNode { u32 count; u16 parent; u8 byte; u8 nbBits; };
struct SymTT { int deltaFindState; u32 deltaNbBits; };
struct FseCT { u32 tableLog; u16 stateTable[512]; SymTT tt[64]; };
struct EncShared {
    u32 count[256];
    // The Huffman stage of a frame is finished before its sequence tables are built, so the Huffman scratch (tree
    // nodes, rank tables, code table, weights) and the OF / ML sequence tables share storage: 9.3 KB per warp
    // instead of 12.4 KB, i.e. 24 instead of 16 resident warps per SM for k_entropy.
    union {
        struct {
            HNode node[2 * 256 + 2];
            u16 rankBase[192], rankCurr[192];
            u8 hufBits[256]; u16 hufCode[256];
            u8 weights[256];
        };
        FseCT ctSeq[2];      // OF, ML
    };
    i16 norm[64];
    u16 cumul[66];
    u8 tableSymbol[512];
    FseCT ct0;              // LL (also borrowed for the Huffman-weight table)
    u32 streamBits[4];
    u32 tmp[8];
    ZB_HD FseCT& ctab(u32 t) { return t == 0 ? ct0 : ctSeq[t - 1]; }
};

// ---- hashing / matching (N/compress/zstd_compress_internal.h:854-945)
ZB_HD u32 hash_ptr(const u8* p, u32 hBits, u32 mls) {
    switch (mls) {
    default:
    case 4: return (load32(p) * 2654435761U) >> (32 - hBits);
    case 5: return (u32)(((load64(p) << 24) * 889523592379ULL) >> (64 - hBits));
    case 6: return (u32)(((load64(p) << 16) * 227718039650203ULL) >> (64 - hBits));
    case 7: return (u32)(((load64(p) << 8) * 58295818150454627ULL) >> (64 - hBits));
    case 8: return (u32)((load64(p) * 0xCF1BBCDCB7A56463ULL) >> (64 - hBits));
    }
}
// ZSTD_count: common prefix of in[] / match[] with in bounded by end
ZB_HD u32 count_match(const u8* in, const u8* match, const u8* end) {
    const u8* const s = in;
    while (in + 8 <= end) {
        u64 const d = load64(in) ^ load64(match);
        if (d) return (u32)(in - s) + (ctz64(d) >> 3);
        in += 8; match += 8;
    }
    while (in < end && *in == *match) { in++; match++; }
    return (u32)(in - s);
}

// ZSTD_compressBlock_doubleFast_noDict_generic, zstd_double_fast.c:105-323, for a fresh frame:
// index = position + 2, zero cells are empty, prefixLowestIndex = 2.  Serial (call from one lane).
// Emits sequences into W.seq* and returns their count; *lastLL gets the trailing literal run.
ZB_HDN u32 parse_dfast(const EncWork& W, const u8* src, size_t srcSize, u32 hBitsL, u32 hBitsS, u32 mls, u32* lastLL) {
    u32* const hashLong = W.hashLong; u32* const hashSmall = W.hashSmall;
    const u8* const base = src - 2;
    const u8* const iend = src + srcSize;
    const u8* const ilimit = iend - 8;
    const u8* const prefixLowest = src;
    const u8* anchor = src;
    const u8* ip = src + 1;                                  // ip += (ip == prefixLowest)
    u32 offset_1 = 1, offset_2 = 4;                          // repStartValue {1,4,8}
    u32 nbSeq = 0;
    {   u32 const maxRep = 1;                                // current - windowLow at position 1
        if (offset_2 > maxRep) offset_2 = 0;
        if (offset_1 > maxRep) offset_1 = 0;
    }
    for (;;) {
        u32 step = 1; const u8* nextStep = ip + 256; const u8* ip1 = ip + step;
        u32 hl0, hl1 = 0, mLength, idxl0, idxl1 = 0, curr = 0, offset = 0;
        const u8* match = nullptr;
        int kind = 0;   // 1 = repcode at ip+1, 2 = long at ip, 3 = short at ip
        if (ip1 > ilimit) break;
        hl0 = hash_ptr(ip, hBitsL, 8); idxl0 = hashLong[hl0];
        for (;;) {
            u32 const hs0 = hash_ptr(ip, hBitsS, mls);
            u32 const idxs0 = hashSmall[hs0];
            curr = (u32)(ip - base);
            hashLong[hl0] = curr; hashSmall[hs0] = curr;
            if ((offset_1 > 0) && (load32(ip + 1 - offset_1) == load32(ip + 1))) { kind = 1; break; }
            hl1 = hash_ptr(ip1, hBitsL, 8);
            if (idxl0 >= 2 && load64(base + idxl0) == load64(ip)) { kind = 2; break; }
            idxl1 = hashLong[hl1];
            if (idxs0 >= 2 && load32(base + idxs0) == load32(ip)) { match = base + idxs0; kind = 3; break; }
            if (ip1 >= nextStep) { step++; nextStep += 256; }
            ip = ip1; ip1 += step;
            hl0 = hl1; idxl0 = idxl1;
            if (ip1 > ilimit) break;
        }
        if (kind == 0) break;
        if (kind == 1) {
            mLength = count_match(ip + 1 + 4, ip + 1 + 4 - offset_1, iend) + 4;
            ip++;
            W.put(nbSeq, (u32)(ip - anchor), 1, mLength); nbSeq++;
        } else {
            if (kind == 2) {
                match = base + idxl0;
                mLength = count_match(ip + 8, match + 8, iend) + 8;
                offset = (u32)(ip - match);
            } else {
                mLength = count_match(ip + 4, match + 4, iend) + 4;
                offset = (u32)(ip - match);
                if ((idxl1 > 2) && (load64(base + idxl1) == load64(ip1))) {
                    const u8* const matchl1 = base + idxl1;
                    u32 const l1len = count_match(ip1 + 8, matchl1 + 8, iend) + 8;
                    if (l1len > mLength) { ip = ip1; mLength = l1len; offset = (u32)(ip - matchl1); match = matchl1; }
                }
            }
            while (((ip > anchor) & (match > prefixLowest)) && (ip[-1] == match[-1])) { ip--; match--; mLength++; }
            offset_2 = offset_1; offset_1 = offset;
            if (step < 4) hashLong[hl1] = (u32)(ip1 - base);
            W.put(nbSeq, (u32)(ip - anchor), offset + 3, mLength); nbSeq++;
        }
        ip += mLength; anchor = ip;
        if (ip <= ilimit) {
            u32 const ins = curr + 2;
            hashLong[hash_ptr(base + ins, hBitsL, 8)] = ins;
            hashLong[hash_ptr(ip - 2, hBitsL, 8)] = (u32)(ip - 2 - base);
            hashSmall[hash_ptr(base + ins, hBitsS, mls)] = ins;
            hashSmall[hash_ptr(ip - 1, hBitsS, mls)] = (u32)(ip - 1 - base);
            while ((ip <= ilimit) && (offset_2 > 0) && (load32(ip) == load32(ip - offset_2))) {
                u32 const rLength = count_match(ip + 4, ip + 4 - offset_2, iend) + 4;
                u32 const t = offset_2; offset_2 = offset_1; offset_1 = t;
                hashSmall[hash_ptr(ip, hBitsS, mls)] = (u32)(ip - base);
                hashLong[hash_ptr(ip, hBitsL, 8)] = (u32)(ip - base);
                W.put(nbSeq, 0, 1, rLength); nbSeq++;
                ip += rLength; anchor = ip;
            }
        }
    }
    *lastLL = (u32)(iend - anchor);
    return nbSeq;
}

// ---------------------------------------------------------------------------------------------
// Warp-cooperative dfast parser (W = 32).  Produces exactly the sequences of parse_dfast() above.
//
// The greedy parse is a chain of decisions, but between two matches the reference just walks
// positions ip, ip+step, ... doing, per position: hash, two table reads, two table writes and up to
// three candidate compares.  A batch of consecutive positions is evaluated by consecutive lanes at
// once.  What lane j must observe is the table as left by positions < j: lanes forward their own
// pending writes to later lanes with __match_any_sync (same slot => the closest earlier lane wins),
// the first lane that finds a match ends the batch, and only lanes up to it commit their writes
// (last writer per slot).  Match extension and the backward catch-up are ballots over 8-byte /
// 1-byte compares.  The batch width adapts (4 -> 32) so that match-dense data does not pay for 32
// speculative probes per sequence.
ZB_HD u32 hash8v(u64 d, u32 hBits) { return (u32)((d * 0xCF1BBCDCB7A56463ULL) >> (64 - hBits)); }
ZB_HD u32 hashSv(u64 d, u32 hBits, u32 mls) {
    switch (mls) {
    default:
    case 4: return ((u32)d * 2654435761U) >> (32 - hBits);
    case 5: return (u32)(((d << 24) * 889523592379ULL) >> (64 - hBits));
    case 6: return (u32)(((d << 16) * 227718039650203ULL) >> (64 - hBits));
    case 7: return (u32)(((d << 8) * 58295818150454627ULL) >> (64 - hBits));
    }
}
// Private table cell of the cooperative parser: index (position + 2, < 2^18) | 14-bit fingerprint << 18 of the bytes
// the reference would compare at that position (8 for the long table, 4 for the short one).  A fingerprint mismatch
// proves the compare would fail, so the candidate bytes -- a random 32-byte HBM sector -- are not fetched at all;
// decisions are unchanged.  Zero still means "empty".
constexpr u32 CELL_IDX_MASK = 0x3FFFF;
// the long table's fingerprint: the 14 bits of the hash product right below the bucket bits (no second multiplication)
ZB_HD u32 tag8(u64 d, u32 hBits) { return (u32)((d * 0xCF1BBCDCB7A56463ULL) >> (50 - hBits)) & 0x3FFFu; }
ZB_HD u32 tag4(u32 d) { return (d * 2246822519U) >> 18; }
ZB_HD u32 cell(u32 idx, u32 tag) { return idx | (tag << 18); }

#ifdef ZB_STATS      // host-only instrumentation (tests/hostsim builds): how much of the speculative work is useful
// Input-stream counters (dfast): coldHeads = batches whose input loads reach a 32-byte sector beyond everything read
// forward so far in the frame; wcReads / wcCold = wcount rounds and those reaching past that mark; near[k] = candidate and
// repcode fetches at an offset below 1 / 2 / 4 / 6 KB / further (k = 0..4).
struct ParseStats { unsigned long long batches, probes, useful, candL, candS, matches, bytes, frames, coldHeads, wcReads, wcCold, near[5]; };
static ParseStats g_parseStats;
static u32 g_statFwd;          // highest input byte + 1 read forward in the current frame
static void stat_fwd(u32 end) { if (end > g_statFwd) g_statFwd = end; }
static void stat_off(u32 off) { g_parseStats.near[off < 1024 ? 0 : off < 2048 ? 1 : off < 4096 ? 2 : off < 6144 ? 3 : 4]++; }
#define ZB_STAT(x) x
#else
#define ZB_STAT(x)
#endif

// common prefix length of src[a..n) and src[b..) (b < a), all lanes cooperate; uniform result
template <class C>
ZB_HD u32 wcount(const C& w, const u8* src, u32 n, u32 a, u32 b) {
    u32 total = 0;
    u32 lanes = C::W < 8 ? C::W : 8;     // most matches are short: start with 64 bytes, then full width
    u32 const lane = lane_of(w);
    for (;;) {
        u32 const pa = a + total + 8u * lane;
        bool const on = lane < lanes;
        u32 const avail = (on && pa < n) ? (n - pa < 8 ? n - pa : 8) : 0;
        u32 cnt = 0;
        if (avail) {
            u64 const da = load64_n(src + pa, avail), db = load64_n(src + (b + total + 8u * lane), avail);
            u64 diff = da ^ db;
            if (avail < 8) diff &= (1ull << (avail * 8)) - 1;
            cnt = diff ? (ctz64(diff) >> 3) : avail;
        }
        ZB_STAT(if (lane == 0) { u32 const e = a + total + 8 * lanes; g_parseStats.wcReads++; g_parseStats.wcCold += e > ((g_statFwd + 31) & ~31u); stat_fwd(e < n ? e : n); })
        u32 const notFull = w.ballot(!on || cnt < 8) & ((lanes >= 32) ? 0xFFFFFFFFu : ((1u << lanes) - 1));
        if (notFull) {
            u32 const f = ctz32(notFull);
            return total + 8 * f + w.shfl(cnt, (int)f);
        }
        total += 8 * lanes;
        lanes = C::W;
    }
}
// backward extension: how many bytes before (ip, m) are equal, limited by maxBack; uniform result
template <class C>
ZB_HD u32 wcatchup(const C& w, const u8* src, u32 ip, u32 m, u32 maxBack) {
    u32 total = 0;
    u32 const lane = lane_of(w);
    for (;;) {
        u32 const k = total + lane;
        bool const eq = (k < maxBack) && (src[ip - 1 - k] == src[m - 1 - k]);
        u32 const mask = w.ballot(eq);
        if (mask != C::FULL) return total + ctz32(~mask);
        total += C::W;
    }
}

// MLS != 0: the short table's match length is known at compile time (level 3's row has 5), so its hash is one expression, no switch
template <class C, u32 MLS = 0>
ZB_HDN u32 parse_dfast_warp(const C& w, const EncWork& W, const u8* src, size_t srcSize, u32 hBitsL, u32 hBitsS, u32 mlsArg, u32* lastLL) {
    u32 const mls = MLS ? MLS : mlsArg;
    u32* const hashLong = W.hashLong; u32* const hashSmall = W.hashSmall;
    int const n = (int)srcSize, ilimit = n - 8;
    int ip = 1, anchor = 0;
    u32 off1 = 1, off2 = 0;             // {1,4,8} clipped by maxRep = 1 at position 1 (zstd_double_fast.c:158-164)
    u32 nbSeq = 0;
    u32 const lane = lane_of(w);
    bool rep2Pending = false;           // the "immediate repcode" test of :308-320 is due at ip (folded into the next batch)
    // Every speculative probe costs ~200 B of random HBM traffic (two table sectors read and written back, two or
    // three candidate sectors), and probes behind the first hit are wasted.  The first batch of a search phase is
    // therefore sized from a running estimate of how many positions recent phases needed; it doubles on a miss.
    u32 est4 = 4 * 3;                   // estimate x4 (fixed point)
    ZB_STAT(if (lane == 0) { g_statFwd = 0; g_parseStats.frames++; })
    for (;;) {   // one iteration per stored match
        u32 step = 1; int nextStep = ip + 256, ip1 = ip + 1;
        if (ip1 > ilimit) {
            // no search position left; the immediate-repcode loop may still fire at ip == ilimit
            while (rep2Pending && (ip <= ilimit) && (off2 > 0) && (load32(src + ip) == load32(src + ip - (int)off2))) {
                u32 const rLength = wcount(w, src, (u32)n, (u32)ip + 4, (u32)ip + 4 - off2) + 4;
                u32 const t = off2; off2 = off1; off1 = t;
                if (lane == 0) { W.put(nbSeq, 0, 1, rLength); }   // table writes are never read again
                nbSeq++; ip += (int)rLength; anchor = ip;
            }
            break;
        }
        u32 width;        // smallest power of two >= the estimate, at most the warp
        {   u32 const want = (est4 + 3) / 4;
            width = want <= 1 ? 1u : (1u << (highbit32(want - 1) + 1));
            if (width > (u32)C::W) width = (u32)C::W; }
        u32 runPos = 0;                   // positions searched in this phase
        int ev = -1;                      // event lane
        // values of the batch that found the event (per lane)
        int p = 0, p1 = 0; u32 st = 1; int ns = 0; u64 d8 = 0; u32 hl = 0, idxl = 0, idxs = 0, kind = 0, nActive = 0; bool plausL = false;
        for (;;) {   // batches of `width` consecutive search positions
            p = ip; p1 = ip1; st = step; ns = nextStep;
            if (step == 1 && ip + (int)width + 1 < nextStep) { p = ip + (int)lane; p1 = p + 1; }
            else for (u32 j = 0; j < lane && j < width; j++) { if (p1 >= ns) { st++; ns += 256; } p = p1; p1 += (int)st; }
            bool const active = lane < width && p1 <= ilimit;
            d8 = active ? load64(src + p) : 0;
            hl = hash8v(d8, hBitsL);
            u32 const hs = hashSv(d8, hBitsS, mls);
            u32 const tl = active ? ld_probe32(hashLong + hl) : 0, ts = active ? ld_probe32(hashSmall + hs) : 0;
            u32 const myTagL = tag8(d8, hBitsL), myTagS = tag4((u32)d8);
            // lane 0 sits at ip: fold the immediate-repcode test into this batch (its load overlaps the table loads)
            bool const rep2Hit = rep2Pending && lane == 0 && off2 > 0 && (load32(src + p - (int)off2) == (u32)d8);
            u32 const mL = w.match_any(active ? hl : (0x80000000u | lane));
            u32 const mS = w.match_any(active ? hs : (0x80000000u | lane));
            u32 const below = (1u << lane) - 1;
            u32 const lowL = mL & below, lowS = mS & below;
            int const pL = w.shfl(p, lowL ? (int)highbit32(lowL) : (int)lane);
            int const pS = w.shfl(p, lowS ? (int)highbit32(lowS) : (int)lane);
            idxl = lowL ? (u32)pL + 2 : (tl & CELL_IDX_MASK);
            idxs = lowS ? (u32)pS + 2 : (ts & CELL_IDX_MASK);
            // candidates forwarded from an earlier lane are a few bytes away (cached); table candidates are only
            // worth a fetch when their fingerprint matches
            plausL = idxl >= 2 && (lowL || (tl >> 18) == myTagL);
            bool const plausS = idxs >= 2 && (lowS || (ts >> 18) == myTagS);
            kind = 0;
            if (active) {
                bool const repOk = (off1 > 0) && (load32(src + p + 1 - (int)off1) == (u32)(d8 >> 8));
                bool const longOk = plausL && (load64(src + (idxl - 2)) == d8);
                bool const shortOk = plausS && (load32(src + (idxs - 2)) == (u32)d8);
                ZB_STAT(g_parseStats.probes++; g_parseStats.candL += plausL && !lowL; g_parseStats.candS += plausS && !lowS;
                        if (off1 > 0) stat_off(off1); if (plausL) stat_off((u32)p + 2 - idxl); if (plausS) stat_off((u32)p + 2 - idxs);
                        if (rep2Pending && lane == 0 && off2 > 0) stat_off(off2);)
                kind = rep2Hit ? 4 : repOk ? 1 : longOk ? 2 : shortOk ? 3 : 0;
            }
            u32 const hm = w.ballot(kind != 0);
            nActive = popc32(w.ballot(active));
            ev = hm ? (int)ctz32(hm) : -1;
            int const last = ev >= 0 ? ev : (int)nActive - 1;
            ZB_STAT({ u32 const e = (u32)w.shfl(p, (int)nActive - 1) + 8;
                      if (lane == 0) { g_parseStats.coldHeads += e > ((g_statFwd + 31) & ~31u); stat_fwd(e < (u32)n ? e : (u32)n); } })
            if (active && (int)lane <= last) {
                u32 const later = ((last >= 31) ? 0xFFFFFFFFu : ((2u << last) - 1)) & ~((2u << lane) - 1);
                if (!(mL & later)) hashLong[hl] = cell((u32)p + 2, myTagL);
                if (!(mS & later)) hashSmall[hs] = cell((u32)p + 2, myTagS);
            }
            w.sync();
            rep2Pending = false;
            runPos += (ev >= 0) ? (u32)ev + 1 : nActive;
            ZB_STAT(if (lane == 0) { g_parseStats.batches++; g_parseStats.useful += (ev >= 0) ? (u32)ev + 1 : nActive; })
            if (ev >= 0) break;
            // no match in this batch: continue after its last position
            {   int const L = (int)nActive - 1;
                int np = p, np1 = p1; u32 nst = st; int nns = ns;
                if (np1 >= nns) { nst++; nns += 256; }
                np = np1; np1 += (int)nst;
                ip = w.shfl(np, L); ip1 = w.shfl(np1, L); step = w.shfl(nst, L); nextStep = w.shfl(nns, L); }
            if (ip1 > ilimit) break;
            width = width * 2 < (u32)C::W ? width * 2 : (u32)C::W;
        }
        if (ev < 0) break;
        est4 = (3 * est4 + 4 * (runPos < 64 ? runPos : 64)) / 4;
        // ---- event at lane ev: gather what the serial code would hold at this point
        u32 const kinde = w.shfl(kind, ev);
        if (kinde == 4) {   // immediate repcode at ip (lane 0): :308-320; its table writes were lane 0's commits
            u32 const rLength = wcount(w, src, (u32)n, (u32)ip + 4, (u32)ip + 4 - off2) + 4;
            u32 const t = off2; off2 = off1; off1 = t;
            if (lane == 0) { W.put(nbSeq, 0, 1, rLength); }
            nbSeq++; ip += (int)rLength; anchor = ip;
            rep2Pending = true;
            continue;
        }
        int const pe = w.shfl(p, ev), p1e = w.shfl(p1, ev);
        u32 const ste = w.shfl(st, ev), idxle = w.shfl(idxl, ev), idxse = w.shfl(idxs, ev);
        bool const nextInBatch = (ev + 1 < (int)nActive);
        int const nl = nextInBatch ? ev + 1 : ev;
        u32 hl1 = w.shfl(hl, nl), idxl1 = w.shfl(idxl, nl); u64 d81 = w.shfl(d8, nl); bool plaus1 = w.shfl((u32)plausL, nl) != 0;
        if (kinde != 1 && !nextInBatch) {   // position ip1 was not part of the batch: read it now (tables are committed)
            d81 = load64(src + p1e); hl1 = hash8v(d81, hBitsL);
            u32 const c1 = ld_probe32(hashLong + hl1); idxl1 = c1 & CELL_IDX_MASK; plaus1 = idxl1 >= 2 && (c1 >> 18) == tag8(d81, hBitsL);
        }
        u32 mLength, offset = 0; int mpos;
        if (kinde == 1) {
            ip = pe + 1;
            mLength = wcount(w, src, (u32)n, (u32)ip + 4, (u32)ip + 4 - off1) + 4;
            if (lane == 0) { W.put(nbSeq, (u32)(ip - anchor), 1, mLength); }
            nbSeq++;
        } else {
            ip = pe;
            if (kinde == 2) {
                mpos = (int)idxle - 2;
                mLength = wcount(w, src, (u32)n, (u32)ip + 8, (u32)mpos + 8) + 8;
                offset = (u32)(ip - mpos);
            } else {
                mpos = (int)idxse - 2;
                mLength = wcount(w, src, (u32)n, (u32)ip + 4, (u32)mpos + 4) + 4;
                offset = (u32)(ip - mpos);
                if ((idxl1 > 2) && plaus1 && (load64(src + (idxl1 - 2)) == d81)) {
                    int const m1 = (int)idxl1 - 2;
                    u32 const l1len = wcount(w, src, (u32)n, (u32)p1e + 8, (u32)m1 + 8) + 8;
                    if (l1len > mLength) { ip = p1e; mLength = l1len; offset = (u32)(ip - m1); mpos = m1; }
                }
            }
            {   u32 const maxBack = (u32)(ip - anchor) < (u32)mpos ? (u32)(ip - anchor) : (u32)mpos;
                u32 const back = maxBack ? wcatchup(w, src, (u32)ip, (u32)mpos, maxBack) : 0;
                ip -= (int)back; mLength += back; }
            off2 = off1; off1 = offset;
            if (lane == 0) {
                if (ste < 4) hashLong[hl1] = cell((u32)p1e + 2, tag8(d81, hBitsL));
                W.put(nbSeq, (u32)(ip - anchor), offset + 3, mLength);
            }
            nbSeq++;
        }
        ip += (int)mLength; anchor = ip;
        if (ip <= ilimit) {
            if (lane == 0) {   // complementary insertions, in the reference's order (:297-305)
                u32 const A = (u32)pe + 2;
                u64 const dA = load64(src + A), dB = load64(src + ip - 2), dC = load64(src + ip - 1);
                hashLong[hash8v(dA, hBitsL)] = cell(A + 2, tag8(dA, hBitsL));
                hashLong[hash8v(dB, hBitsL)] = cell((u32)ip - 2 + 2, tag8(dB, hBitsL));
                hashSmall[hashSv(dA, hBitsS, mls)] = cell(A + 2, tag4((u32)dA));
                hashSmall[hashSv(dC, hBitsS, mls)] = cell((u32)ip - 1 + 2, tag4((u32)dC));
            }
            rep2Pending = true;
        }
        w.sync();
    }
    w.sync();
    ZB_STAT(if (lane == 0) { g_parseStats.matches += nbSeq; g_parseStats.bytes += (unsigned long long)n; })
    *lastLL = (u32)(n - anchor);
    return nbSeq;
}

// ---- forward bit writer (LSB first); close appends the 1-bit end mark.
// Mirrors BIT_CStream_t / HUF_CStream_t bounds: 8 bytes of slack are required (bitstream.h:226-242).
struct BitW {
    u8* p; size_t cap; size_t n; u64 acc; u32 nb;
    ZB_HD void init(u8* dst, size_t c) { p = dst; cap = c; n = 0; acc = 0; nb = 0; }
    ZB_HD void add(u64 v, u32 bits) {
        if (!bits) return;
        v &= (bits >= 64) ? ~0ull : ((1ull << bits) - 1);
        acc |= v << nb; nb += bits;
        while (nb >= 8) { if (n < cap) p[n] = (u8)acc; n++; acc >>= 8; nb -= 8; }
    }
    ZB_HD size_t flush_partial() { if (nb) { if (n < cap) p[n] = (u8)acc; n++; acc = 0; nb = 0; } return n; }
    ZB_HD size_t close() {
        add(1, 1);
        if (cap <= 8 || n >= cap - 8) return 0;
        if (nb) { p[n] = (u8)acc; return n + 1; }
        return n;
    }
};

// ---- cooperative bit packing: every lane appends the bits of its own slice of a stream at a bit offset
// obtained from a prefix sum over the slice sizes.  The region is zeroed first; bytes a lane fully owns are
// plain stores, the (at most two) bytes it shares with its neighbours are OR-ed in atomically.
template <class C>
struct LaneBits {
    u8* base; u32 bytePos; u64 acc; u32 nb; bool shared;
    ZB_HD void init(u8* b, u32 startBit) { base = b; bytePos = startBit >> 3; nb = startBit & 7; acc = 0; shared = nb != 0; }
    ZB_HD void emit(const C& w) {          // write all whole bytes held in acc
        // interior of the lane's region: one aligned 32-bit store instead of four byte stores (a byte store per lane is
        // a separate sector write at L2)
        if (!shared && nb >= 32 && ((reinterpret_cast<uintptr_t>(base) + bytePos) & 3) == 0) {
            *reinterpret_cast<u32*>(base + bytePos) = (u32)acc;
            bytePos += 4; acc >>= 32; nb -= 32;
        }
        while (nb >= 8) {
            if (shared) { w.atomic_or_byte(base + bytePos, (u32)(acc & 0xFF)); shared = false; }
            else base[bytePos] = (u8)acc;
            bytePos++; acc >>= 8; nb -= 8;
        }
    }
    ZB_HD void add(const C& w, u32 v, u32 bits) {   // bits <= 31; v must fit in `bits`
        acc |= (u64)v << nb; nb += bits;
        if (nb >= 32) emit(w);
    }
    ZB_HD void close(const C& w) { emit(w); if (nb) w.atomic_or_byte(base + bytePos, (u32)(acc & 0xFF)); }
};

// ---- warp histogram of bytes; returns largest count, trims *maxSV (HIST_count_simple, hist.c:39-74)
template <class C>
ZB_HDN u32 hist_warp(const C& w, u32* count, u32* maxSV, const u8* src, size_t n) {
    u32 const m0 = *maxSV;
    for (u32 s = (u32)w.lane; s <= m0; s += C::W) count[s] = 0;
    w.sync();
    if (n == 0) { *maxSV = 0; return 0; }
    for (size_t i = (size_t)w.lane; i < n; i += C::W) w.atomic_inc(&count[src[i]]);
    w.sync();
    u32 largest = 0, top = 0;
    for (u32 s = (u32)w.lane; s <= m0; s += C::W) { u32 const c = count[s]; if (c > largest) largest = c; if (c) top = s; }
    largest = w.max(largest); top = w.max(top);
    *maxSV = top;
    return largest;
}
// scalar variant for tiny inputs handled by one lane
ZB_HDN u32 hist_serial(u32* count, u32* maxSV, const u8* src, size_t n) {
    u32 m = *maxSV, largest = 0;
    for (u32 s = 0; s <= m; s++) count[s] = 0;
    if (n == 0) { *maxSV = 0; return 0; }
    for (size_t i = 0; i < n; i++) count[src[i]]++;
    while (!count[m]) m--;
    *maxSV = m;
    for (u32 s = 0; s <= m; s++) if (count[s] > largest) largest = count[s];
    return largest;
}

// ------------------------------------------------------------------- FSE
// FSE_optimalTableLog_internal, fse_compress.c:348-369
ZB_HD u32 fse_optimal_log(u32 maxTableLog, size_t srcSize, u32 maxSV, u32 minus) {
    u32 const maxBitsSrc = highbit32((u32)(srcSize - 1)) - minus;
    u32 tableLog = maxTableLog;
    u32 const minBitsSrc = highbit32((u32)srcSize) + 1, minBitsSymbols = highbit32(maxSV) + 2;
    u32 const minBits = minBitsSrc < minBitsSymbols ? minBitsSrc : minBitsSymbols;
    if (tableLog == 0) tableLog = 11;
    if (maxBitsSrc < tableLog) tableLog = maxBitsSrc;
    if (minBits > tableLog) tableLog = minBits;
    if (tableLog < 5) tableLog = 5;
    if (tableLog > 12) tableLog = 12;
    return tableLog;
}
// FSE_normalizeM2 :379-463
ZB_HDN size_t fse_normalize_m2(i16* norm, u32 tableLog, const u32* count, size_t total, u32 maxSV, i16 lowProbCount) {
    i16 const NOT_YET = -2; u32 distributed = 0, ToDistribute;
    u32 const lowThreshold = (u32)(total >> tableLog);
    u32 lowOne = (u32)((total * 3) >> (tableLog + 1));
    for (u32 s = 0; s <= maxSV; s++) {
        if (count[s] == 0) { norm[s] = 0; continue; }
        if (count[s] <= lowThreshold) { norm[s] = lowProbCount; distributed++; total -= count[s]; continue; }
        if (count[s] <= lowOne) { norm[s] = 1; distributed++; total -= count[s]; continue; }
        norm[s] = NOT_YET;
    }
    ToDistribute = (1u << tableLog) - distributed;
    if (ToDistribute == 0) return 0;
    if ((total / ToDistribute) > lowOne) {
        lowOne = (u32)((total * 3) / (ToDistribute * 2));
        for (u32 s = 0; s <= maxSV; s++)
            if ((norm[s] == NOT_YET) && (count[s] <= lowOne)) { norm[s] = 1; distributed++; total -= count[s]; }
        ToDistribute = (1u << tableLog) - distributed;
    }
    if (distributed == maxSV + 1) {
        u32 maxV = 0, maxC = 0;
        for (u32 s = 0; s <= maxSV; s++) if (count[s] > maxC) { maxV = s; maxC = count[s]; }
        norm[maxV] = (i16)(norm[maxV] + (i16)ToDistribute);
        return 0;
    }
    if (total == 0) {
        for (u32 s = 0; ToDistribute > 0; s = (s + 1) % (maxSV + 1))
            if (norm[s] > 0) { ToDistribute--; norm[s]++; }
        return 0;
    }
    u64 const vStepLog = 62 - tableLog;
    u64 const mid = (1ULL << (vStepLog - 1)) - 1;
    u64 const rStep = ((((u64)1 << vStepLog) * ToDistribute) + mid) / (u32)total;
    u64 tmpTotal = mid;
    for (u32 s = 0; s <= maxSV; s++) {
        if (norm[s] == NOT_YET) {
            u64 const end = tmpTotal + (count[s] * rStep);
            u32 const sStart = (u32)(tmpTotal >> vStepLog), sEnd = (u32)(end >> vStepLog);
            u32 const weight = sEnd - sStart;
            if (weight < 1) return ERR(E_GENERIC);
            norm[s] = (i16)weight; tmpTotal = end;
        }
    }
    return 0;
}
// FSE_normalizeCount :465-525
ZB_HDN size_t fse_normalize(i16* norm, u32 tableLog, const u32* count, size_t total, u32 maxSV, bool useLowProb) {
    const u32 rtb[8] = { 0, 473195, 504333, 520860, 550000, 700000, 750000, 830000 };
    i16 const lowProbCount = useLowProb ? -1 : 1;
    u64 const scale = 62 - tableLog;
    u64 const step = ((u64)1 << 62) / (u32)total;
    u64 const vStep = 1ULL << (scale - 20);
    int still = 1 << tableLog;
    u32 largest = 0; i16 largestP = 0;
    u32 const lowThreshold = (u32)(total >> tableLog);
    if (tableLog < 5) return ERR(E_GENERIC);
    if (tableLog > 12) return ERR(E_tableLog_tooLarge);
    {   u32 const a = highbit32((u32)total) + 1, b = highbit32(maxSV) + 2;
        if (tableLog < (a < b ? a : b)) return ERR(E_GENERIC); }
    for (u32 s = 0; s <= maxSV; s++) {
        if (count[s] == total) return 0;
        if (count[s] == 0) { norm[s] = 0; continue; }
        if (count[s] <= lowThreshold) { norm[s] = lowProbCount; still--; }
        else {
            i16 proba = (i16)((count[s] * step) >> scale);
            if (proba < 8) { u64 const restToBeat = vStep * rtb[proba]; proba = (i16)(proba + (((count[s] * step) - ((u64)proba << scale)) > restToBeat)); }
            if (proba > largestP) { largestP = proba; largest = s; }
            norm[s] = proba; still -= proba;
        }
    }
    if (-still >= (norm[largest] >> 1)) {
        size_t const e = fse_normalize_m2(norm, tableLog, count, total, maxSV, lowProbCount);
        if (isErr(e)) return e;
    } else norm[largest] = (i16)(norm[largest] + (i16)still);
    return tableLog;
}
// FSE_writeNCount_generic :233-327
ZB_HDN size_t fse_write_ncount(u8* dst, size_t cap, const i16* norm, u32 maxSV, u32 tableLog) {
    BitW w; w.init(dst, cap);
    int nbBits, remaining, threshold; bool previousIs0 = false; u32 symbol = 0; u32 const alphabetSize = maxSV + 1;
    int const tableSize = 1 << tableLog;
    w.add(tableLog - 5, 4);
    remaining = tableSize + 1; threshold = tableSize; nbBits = (int)tableLog + 1;
    while ((symbol < alphabetSize) && (remaining > 1)) {
        if (previousIs0) {
            u32 start = symbol;
            while ((symbol < alphabetSize) && !norm[symbol]) symbol++;
            if (symbol == alphabetSize) break;
            while (symbol >= start + 24) { start += 24; w.add(0xFFFF, 16); }
            while (symbol >= start + 3) { start += 3; w.add(3, 2); }
            w.add(symbol - start, 2);
        }
        int count = norm[symbol++];
        int const max = (2 * threshold - 1) - remaining;
        remaining -= count < 0 ? -count : count;
        count++;
        if (count >= threshold) count += max;
        w.add((u64)count, (u32)(nbBits - (count < max)));
        previousIs0 = (count == 1);
        if (remaining < 1) return ERR(E_GENERIC);
        while (remaining < threshold) { nbBits--; threshold >>= 1; }
    }
    if (remaining != 1) return ERR(E_GENERIC);
    size_t const n = w.flush_partial();
    if (n > cap) return ERR(E_dstSize_tooSmall);
    return n;
}
// FSE_buildCTable_wksp :68-214
ZB_HDN void fse_build_ctable(FseCT& ct, const i16* norm, u32 maxSV, u32 tableLog, u16* cumul, u8* tableSymbol) {
    u32 const tableSize = 1u << tableLog, mask = tableSize - 1, step = (tableSize >> 1) + (tableSize >> 3) + 3;
    u32 high = tableSize - 1, pos = 0;
    ct.tableLog = tableLog;
    cumul[0] = 0;
    for (u32 u = 1; u <= maxSV + 1; u++) {
        if (norm[u - 1] == -1) { cumul[u] = (u16)(cumul[u - 1] + 1); tableSymbol[high--] = (u8)(u - 1); }
        else cumul[u] = (u16)(cumul[u - 1] + (u16)norm[u - 1]);
    }
    cumul[maxSV + 1] = (u16)(tableSize + 1);
    for (u32 s = 0; s <= maxSV; s++) {
        int const n = norm[s];
        for (int i = 0; i < n; i++) {
            tableSymbol[pos] = (u8)s;
            pos = (pos + step) & mask;
            while (pos > high) pos = (pos + step) & mask;
        }
    }
    for (u32 u = 0; u < tableSize; u++) { u8 const sy = tableSymbol[u]; ct.stateTable[cumul[sy]++] = (u16)(tableSize + u); }
    u32 total = 0;
    for (u32 s = 0; s <= maxSV; s++) {
        int const n = norm[s];
        if (n == 0) { ct.tt[s].deltaNbBits = ((tableLog + 1) << 16) - (1u << tableLog); ct.tt[s].deltaFindState = 0; }
        else if (n == -1 || n == 1) { ct.tt[s].deltaNbBits = (tableLog << 16) - (1u << tableLog); ct.tt[s].deltaFindState = (int)(total - 1); total++; }
        else {
            u32 const maxBitsOut = tableLog - highbit32((u32)n - 1);
            u32 const minStatePlus = (u32)n << maxBitsOut;
            ct.tt[s].deltaNbBits = (maxBitsOut << 16) - minStatePlus;
            ct.tt[s].deltaFindState = (int)(total - (u32)n);
            total += (u32)n;
        }
    }
}
ZB_HD void fse_build_ctable_rle(FseCT& ct, u32 symbol) { ct.tableLog = 0; ct.stateTable[0] = 0; ct.stateTable[1] = 0; ct.tt[symbol].deltaNbBits = 0; ct.tt[symbol].deltaFindState = 0; }
// FSE_initCState2 / FSE_encodeSymbol, N/common/fse.h:428-461
ZB_HD u32 fse_init_state2(const FseCT& ct, u32 symbol) {
    SymTT const tt = ct.tt[symbol];
    u32 const nbBitsOut = (tt.deltaNbBits + (1 << 15)) >> 16;
    u32 const v = (nbBitsOut << 16) - tt.deltaNbBits;
    return ct.stateTable[(int)(v >> nbBitsOut) + tt.deltaFindState];
}
ZB_HD u32 fse_encode(BitW& w, const FseCT& ct, u32 state, u32 symbol) {
    SymTT const tt = ct.tt[symbol];
    u32 const nbBitsOut = (state + tt.deltaNbBits) >> 16;
    w.add(state, nbBitsOut);
    return ct.stateTable[(int)(state >> nbBitsOut) + tt.deltaFindState];
}

// --------------------------------------------------------------- Huffman
// HUF_sort & friends, huf_compress.c:530-665.  The quicksort is restated operation for
// operation (with an explicit stack): the order it leaves equal counts in decides the codes.
constexpr u32 HUF_LOG_BUCKETS_BEGIN = 158, HUF_DISTINCT_CUTOFF = 165, HUF_RANK_TABLE = 192;
ZB_HD u32 huf_bucket(u32 count) { return count < HUF_DISTINCT_CUTOFF ? count : highbit32(count) + HUF_LOG_BUCKETS_BEGIN; }
ZB_HD void hnode_swap(HNode* a, HNode* b) { HNode const t = *a; *a = *b; *b = t; }
ZB_HDN void huf_insertion(HNode* a, int low, int high) {
    int const size = high - low + 1; a += low;
    for (int i = 1; i < size; i++) { HNode const key = a[i]; int j = i - 1; while (j >= 0 && a[j].count < key.count) { a[j + 1] = a[j]; j--; } a[j + 1] = key; }
}
ZB_HD int huf_partition(HNode* a, int low, int high) {
    u32 const pivot = a[high].count; int i = low - 1;
    for (int j = low; j < high; j++) if (a[j].count > pivot) { i++; hnode_swap(&a[i], &a[j]); }
    hnode_swap(&a[i + 1], &a[high]);
    return i + 1;
}
ZB_HDN void huf_quicksort(HNode* a, int low, int high) {
    // HUF_simpleQuickSort recurses on the smaller side and keeps looping on the larger one.
    // The pending loops are kept on an explicit stack (depth <= log2(256) + 1); a popped frame
    // resumes *inside* its while loop, i.e. without re-testing the insertion-sort threshold.
    int stLo[16], stHi[16]; int sp = 0;
    bool enter = true;
    for (;;) {
        if (enter) {
            if (high - low < 8) { huf_insertion(a, low, high); enter = false; if (sp == 0) return; sp--; low = stLo[sp]; high = stHi[sp]; continue; }
            enter = false;
        }
        if (low < high) {
            int const idx = huf_partition(a, low, high);
            if (idx - low < high - idx) { stLo[sp] = idx + 1; stHi[sp] = high; sp++; high = idx - 1; }
            else { stLo[sp] = low; stHi[sp] = idx - 1; sp++; low = idx + 1; }
            enter = true;
        } else {
            if (sp == 0) return;
            sp--; low = stLo[sp]; high = stHi[sp];
        }
    }
}
ZB_HDN void huf_sort(EncShared& S, const u32* count, u32 maxSV) {
    HNode* const node = S.node + 1;
    for (u32 n = 0; n < HUF_RANK_TABLE; n++) { S.rankBase[n] = 0; S.rankCurr[n] = 0; }
    for (u32 n = 0; n <= maxSV; n++) S.rankBase[huf_bucket(count[n])]++;
    for (u32 n = HUF_RANK_TABLE - 1; n > 0; n--) { S.rankBase[n - 1] = (u16)(S.rankBase[n - 1] + S.rankBase[n]); S.rankCurr[n - 1] = S.rankBase[n - 1]; }
    for (u32 n = 0; n <= maxSV; n++) {
        u32 const c = count[n], r = huf_bucket(c) + 1, pos = S.rankCurr[r]++;
        node[pos].count = c; node[pos].byte = (u8)n;
    }
    for (u32 n = HUF_DISTINCT_CUTOFF; n < HUF_RANK_TABLE - 1; n++) {
        int const bucketSize = (int)S.rankCurr[n] - (int)S.rankBase[n];
        if (bucketSize > 1) huf_quicksort(node + S.rankBase[n], 0, bucketSize - 1);
    }
}
// HUF_setMaxHeight :376-498
ZB_HDN u32 huf_set_max_height(HNode* node, u32 lastNonNull, u32 target) {
    u32 const largestBits = node[lastNonNull].nbBits;
    if (largestBits <= target) return largestBits;
    int totalCost = 0; u32 const baseCost = 1u << (largestBits - target); int n = (int)lastNonNull;
    while (node[n].nbBits > target) { totalCost += (int)(baseCost - (1u << (largestBits - node[n].nbBits))); node[n].nbBits = (u8)target; n--; }
    while (node[n].nbBits == target) --n;
    totalCost >>= (largestBits - target);
    u32 const noSymbol = 0xF0F0F0F0; u32 rankLast[HUF_TABLELOG_MAX + 2];
    for (u32 r = 0; r < HUF_TABLELOG_MAX + 2; r++) rankLast[r] = noSymbol;
    {   u32 currentNbBits = target;
        for (int pos = n; pos >= 0; pos--) {
            if (node[pos].nbBits >= currentNbBits) continue;
            currentNbBits = node[pos].nbBits;
            rankLast[target - currentNbBits] = (u32)pos;
        } }
    while (totalCost > 0) {
        u32 nBitsToDecrease = highbit32((u32)totalCost) + 1;
        for (; nBitsToDecrease > 1; nBitsToDecrease--) {
            u32 const highPos = rankLast[nBitsToDecrease], lowPos = rankLast[nBitsToDecrease - 1];
            if (highPos == noSymbol) continue;
            if (lowPos == noSymbol) break;
            u32 const highTotal = node[highPos].count, lowTotal = 2 * node[lowPos].count;
            if (highTotal <= lowTotal) break;
        }
        while ((nBitsToDecrease <= HUF_TABLELOG_MAX) && (rankLast[nBitsToDecrease] == noSymbol)) nBitsToDecrease++;
        totalCost -= 1 << (nBitsToDecrease - 1);
        node[rankLast[nBitsToDecrease]].nbBits++;
        if (rankLast[nBitsToDecrease - 1] == noSymbol) rankLast[nBitsToDecrease - 1] = rankLast[nBitsToDecrease];
        if (rankLast[nBitsToDecrease] == 0) rankLast[nBitsToDecrease] = noSymbol;
        else {
            rankLast[nBitsToDecrease]--;
            if (node[rankLast[nBitsToDecrease]].nbBits != target - nBitsToDecrease) rankLast[nBitsToDecrease] = noSymbol;
        }
    }
    while (totalCost < 0) {
        if (rankLast[1] == noSymbol) {
            while (node[n].nbBits == target) n--;
            node[n + 1].nbBits--; rankLast[1] = (u32)(n + 1); totalCost++;
            continue;
        }
        node[rankLast[1] + 1].nbBits--; rankLast[1]++; totalCost++;
    }
    return target;
}
// HUF_buildCTable_wksp :755-791 (sort, HUF_buildTree :681-718, setMaxHeight, HUF_buildCTableFromTree :730-753)
ZB_HDN u32 huf_build_ctable(EncShared& S, const u32* count, u32 maxSV, u32 maxNbBits) {
    HNode* const node0 = S.node; HNode* const node = S.node + 1;
    for (u32 i = 0; i < 2 * 256 + 2; i++) { node0[i].count = 0; node0[i].parent = 0; node0[i].byte = 0; node0[i].nbBits = 0; }
    huf_sort(S, count, maxSV);
    int nonNull = (int)maxSV;
    while (node[nonNull].count == 0) nonNull--;
    int lowS = nonNull, nodeNb = 256, lowN = 256; int const nodeRoot = nodeNb + lowS - 1;
    node[nodeNb].count = node[lowS].count + node[lowS - 1].count;
    node[lowS].parent = node[lowS - 1].parent = (u16)nodeNb;
    nodeNb++; lowS -= 2;
    for (int n = nodeNb; n <= nodeRoot; n++) node[n].count = 1u << 30;
    node0[0].count = 1u << 31;
    while (nodeNb <= nodeRoot) {
        int const n1 = (node[lowS].count < node[lowN].count) ? lowS-- : lowN++;
        int const n2 = (node[lowS].count < node[lowN].count) ? lowS-- : lowN++;
        node[nodeNb].count = node[n1].count + node[n2].count;
        node[n1].parent = node[n2].parent = (u16)nodeNb;
        nodeNb++;
    }
    node[nodeRoot].nbBits = 0;
    for (int n = nodeRoot - 1; n >= 256; n--) node[n].nbBits = (u8)(node[node[n].parent].nbBits + 1);
    for (int n = 0; n <= nonNull; n++) node[n].nbBits = (u8)(node[node[n].parent].nbBits + 1);
    maxNbBits = huf_set_max_height(node, (u32)nonNull, maxNbBits);
    u16 nbPerRank[HUF_TABLELOG_MAX + 1], valPerRank[HUF_TABLELOG_MAX + 1];
    for (u32 r = 0; r <= HUF_TABLELOG_MAX; r++) { nbPerRank[r] = 0; valPerRank[r] = 0; }
    for (int n = 0; n <= nonNull; n++) nbPerRank[node[n].nbBits]++;
    {   u16 min = 0;
        for (int n = (int)maxNbBits; n > 0; n--) { valPerRank[n] = min; min = (u16)(min + nbPerRank[n]); min >>= 1; } }
    for (u32 n = 0; n <= maxSV; n++) S.hufBits[node[n].byte] = node[n].nbBits;
    for (u32 n = 0; n <= maxSV; n++) S.hufCode[n] = S.hufBits[n] ? valPerRank[S.hufBits[n]]++ : 0;
    return maxNbBits;
}
// FSE_compress_usingCTable_generic :551-608
ZB_HDN size_t fse_compress_2states(u8* dst, size_t cap, const u8* src, size_t srcSize, const FseCT& ct) {
    const u8* ip = src + srcSize; BitW w; u32 s1, s2;
    if (srcSize <= 2) return 0;
    if (cap <= 8) return 0;
    w.init(dst, cap);
    if (srcSize & 1) { s1 = fse_init_state2(ct, *--ip); s2 = fse_init_state2(ct, *--ip); s1 = fse_encode(w, ct, s1, *--ip); }
    else { s2 = fse_init_state2(ct, *--ip); s1 = fse_init_state2(ct, *--ip); }
    srcSize -= 2;
    if (srcSize & 2) { s2 = fse_encode(w, ct, s2, *--ip); s1 = fse_encode(w, ct, s1, *--ip); }
    while (ip > src) {
        s2 = fse_encode(w, ct, s2, *--ip); s1 = fse_encode(w, ct, s1, *--ip);
        s2 = fse_encode(w, ct, s2, *--ip); s1 = fse_encode(w, ct, s1, *--ip);
    }
    w.add(s2, ct.tableLog); w.add(s1, ct.tableLog);
    return w.close();
}
// HUF_writeCTable_wksp :248-289 (+ HUF_compressWeights :146-186); lane 0
ZB_HDN size_t huf_write_ctable(EncShared& S, u8* dst, size_t cap, u32 maxSV, u32 huffLog) {
    u8* const wt = S.weights;
    for (u32 n = 0; n < maxSV; n++) wt[n] = S.hufBits[n] ? (u8)(huffLog + 1 - S.hufBits[n]) : 0;
    if (cap < 1) return ERR(E_dstSize_tooSmall);
    size_t hSize = 0;
    do {   // HUF_compressWeights(dst+1, cap-1, wt, maxSV)
        u8* const o = dst + 1; size_t const ocap = cap - 1; size_t const wtSize = maxSV;
        if (wtSize <= 1) { hSize = 0; break; }
        u32 cnt[HUF_TABLELOG_MAX + 1]; u32 m = HUF_TABLELOG_MAX;
        u32 const maxCount = hist_serial(cnt, &m, wt, wtSize);
        if (maxCount == wtSize) { hSize = 1; break; }
        if (maxCount == 1) { hSize = 0; break; }
        u32 const tableLog = fse_optimal_log(6, wtSize, m, 2);
        i16 norm[HUF_TABLELOG_MAX + 1];
        {   size_t const e = fse_normalize(norm, tableLog, cnt, wtSize, m, false); if (isErr(e)) { hSize = e; break; } }
        size_t const h = fse_write_ncount(o, ocap, norm, m, tableLog);
        if (isErr(h)) { hSize = h; break; }
        fse_build_ctable(S.ctab(0), norm, m, tableLog, S.cumul, S.tableSymbol);
        size_t const c = fse_compress_2states(o + h, ocap - h, wt, wtSize, S.ctab(0));
        if (c == 0) { hSize = 0; break; }
        hSize = h + c;
    } while (0);
    if (isErr(hSize)) return hSize;
    if ((hSize > 1) & (hSize < maxSV / 2)) { dst[0] = (u8)hSize; return hSize + 1; }
    if (maxSV > 128) return ERR(E_GENERIC);
    if (((maxSV + 1) / 2) + 1 > cap) return ERR(E_dstSize_tooSmall);
    dst[0] = (u8)(128 + (maxSV - 1));
    wt[maxSV] = 0;
    for (u32 n = 0; n < maxSV; n += 2) dst[(n / 2) + 1] = (u8)((wt[n] << 4) + wt[n + 1]);
    return ((maxSV + 1) / 2) + 1;
}
// one Huffman stream (HUF_compress1X_usingCTable_internal_body :1055-1118): symbols are appended last-to-first
// (LSB first), then a single 1 bit.  The whole group packs it: lane l takes the l-th slice of the emission
// order, slice bit offsets come from an exclusive scan.  `totalBits` = sum of code lengths (without the mark).
// Returns the stream size in bytes, 0 when it does not fit (same bounds as HUF_closeCStream :973-982).
template <class C>
ZB_HDN size_t huf_encode_stream(const C& w, const EncShared& S, u8* dst, size_t cap, const u8* src, size_t n, u32 totalBits) {
    if (cap <= 8) return 0;
    if ((((size_t)totalBits + 1) >> 3) >= cap - 8) return 0;
    size_t const size = ((size_t)totalBits + 1 + 7) >> 3;
    for (size_t i = (size_t)w.lane; i < size; i += C::W) dst[i] = 0;
    w.sync();
    u32 const B = (u32)((n + C::W - 1) / C::W);
    u32 const j0 = (u32)w.lane * B < (u32)n ? (u32)w.lane * B : (u32)n;
    u32 const j1 = j0 + B < (u32)n ? j0 + B : (u32)n;
    // every lane walks its own slice, so byte loads would be 32 separate sector requests per instruction and eight
    // of them per sector: read the slice eight symbols at a time instead
    u32 mine = 0;
    for (u32 j = j0; j < j1;) {
        u32 const cnt = j1 - j < 8 ? j1 - j : 8;
        u64 const v = load64_n(src + (n - j - cnt), cnt);
        for (u32 k = 0; k < cnt; k++) mine += S.hufBits[(u8)(v >> (8 * (cnt - 1 - k)))];
        j += cnt;
    }
    u32 const start = w.exscan(mine);
    LaneBits<C> lb; lb.init(dst, start);
    for (u32 j = j0; j < j1;) {
        u32 const cnt = j1 - j < 8 ? j1 - j : 8;
        u64 const v = load64_n(src + (n - j - cnt), cnt);
        for (u32 k = 0; k < cnt; k++) { u8 const b = (u8)(v >> (8 * (cnt - 1 - k))); lb.add(w, S.hufCode[b], S.hufBits[b]); }
        j += cnt;
    }
    if (w.lane == C::W - 1) lb.add(w, 1, 1);
    lb.close(w);
    w.sync();
    return size;
}

// ZSTD_noCompressLiterals :39-66 / ZSTD_compressRleLiteralsBlock :81-107 ; warp copy
template <class C>
ZB_HDN size_t lit_raw(const C& w, u8* dst, size_t cap, const u8* src, size_t n) {
    u32 const fl = 1 + (n > 31) + (n > 4095);
    if (n + fl > cap) return ERR(E_dstSize_tooSmall);
    if (w.lane == 0) {
        if (fl == 1) dst[0] = (u8)(n << 3);
        else if (fl == 2) { u32 const v = (1 << 2) + (u32)(n << 4); dst[0] = (u8)v; dst[1] = (u8)(v >> 8); }
        else { u32 const v = (3 << 2) + (u32)(n << 4); dst[0] = (u8)v; dst[1] = (u8)(v >> 8); dst[2] = (u8)(v >> 16); }
    }
    wcopy(w, dst + fl, src, n);
    w.sync();
    return n + fl;
}
template <class C>
ZB_HDN size_t lit_rle(const C& w, u8* dst, const u8* src, size_t n) {
    u32 const fl = 1 + (n > 31) + (n > 4095);
    if (w.lane == 0) {
        if (fl == 1) dst[0] = (u8)(1 + (n << 3));
        else if (fl == 2) { u32 const v = 1 + (1 << 2) + (u32)(n << 4); dst[0] = (u8)v; dst[1] = (u8)(v >> 8); }
        else { u32 const v = 1 + (3 << 2) + (u32)(n << 4); dst[0] = (u8)v; dst[1] = (u8)(v >> 8); dst[2] = (u8)(v >> 16); }
        dst[fl] = src[0];
    }
    w.sync();
    return fl + 1;
}

// ZSTD_compressLiterals (zstd_compress_literals.c:129-235) + HUF_compress_internal (huf_compress.c:1332-1434),
// first block of a frame (no previous Huffman table).  Uniform return value.
template <class C>
ZB_HDN size_t compress_literals(const C& w, EncShared& S, u8* dst, size_t cap, const u8* src, size_t n, u32 strategy, bool disableLitCompression, bool suspectUncompressible) {
    size_t const lhSize = 3 + (n >= 1024) + (n >= 16384); bool const single = n < 256;
    ZB_PT_DECL
    if (disableLitCompression) return lit_raw(w, dst, cap, src, n);
    {   int const sh = (9 - (int)strategy) < 3 ? (9 - (int)strategy) : 3;
        if (n < ((size_t)8 << sh)) return lit_raw(w, dst, cap, src, n); }
    if (cap < lhSize + 1) return ERR(E_dstSize_tooSmall);
    u8* const o = dst + lhSize; size_t const ocap = cap - lhSize;
    size_t cLit = 0;   // 0 = not compressible
    do {
        if (!ocap) break;
        if (suspectUncompressible && n >= 4096 * 10) {      // :1367-1379
            u32 m1 = 255, m2 = 255; size_t largestTotal = 0;
            largestTotal += hist_warp(w, S.count, &m1, src, 4096);
            largestTotal += hist_warp(w, S.count, &m2, src + n - 4096, 4096);
            if (largestTotal <= ((2 * 4096) >> 7) + 4) break;
        }
        u32 maxSV = 255;
        u32 const largest = hist_warp(w, S.count, &maxSV, src, n);
        ZB_PT(7);      // literal histogram
        if (largest == n) { if (w.lane == 0) o[0] = src[0]; cLit = 1; break; }
        if (largest <= (n >> 7) + 4) break;
        // tree + table description on lane 0
        size_t hSize = 0; u32 huffLog = 0;
        if (w.lane == 0) {
            huffLog = fse_optimal_log(LitHufLog, n, maxSV, 1);     // HUF_optimalTableLog cheap path :1284-1287
            huffLog = huf_build_ctable(S, S.count, maxSV, huffLog);
            hSize = huf_write_ctable(S, o, ocap, maxSV, huffLog);
        }
        w.sync();
        hSize = w.bcast(hSize);
        ZB_PT(8);      // Huffman tree + table description (lane 0)
        if (isErr(hSize)) { cLit = hSize; break; }
        if (hSize + 12ul >= n) break;
        u8* op = o + hSize; size_t const opcap = ocap - hSize;
        size_t total;
        if (single) {
            u32 b = 0;
            for (size_t i = (size_t)w.lane; i < n; i += C::W) b += S.hufBits[src[i]];
            u32 const bits = w.sum(b);
            size_t const c = huf_encode_stream(w, S, op, opcap, src, n, bits);
            if (c == 0) break;
            total = hSize + c;
        } else {
            // HUF_compress4X_usingCTable_internal :1167-1215
            if (opcap < 6 + 1 + 1 + 1 + 8) break;
            if (n < 12) break;
            size_t const seg = (n + 3) / 4;
            u32 bits[4];
            for (int k = 0; k < 4; k++) {      // sizing pass: bits of each stream, all lanes
                const u8* const sk = src + (size_t)k * seg; size_t const len = (k < 3) ? seg : n - 3 * seg;
                u32 b = 0;
                for (size_t i = (size_t)w.lane; i < len; i += C::W) b += S.hufBits[sk[i]];
                bits[k] = w.sum(b);
            }
            size_t acc = 6; bool fail = false;
            for (int k = 0; k < 4; k++) {
                const u8* const sk = src + (size_t)k * seg; size_t const len = (k < 3) ? seg : n - 3 * seg;
                // the reference encodes stream k into what is left of the buffer and gives up on overflow or > 65535 bytes
                size_t const c = huf_encode_stream(w, S, op + acc, opcap - acc, sk, len, bits[k]);
                if (c == 0 || c > 65535) { fail = true; break; }
                if (k < 3 && w.lane == 0) { op[2 * k] = (u8)c; op[2 * k + 1] = (u8)(c >> 8); }
                acc += c;
            }
            w.sync();
            if (fail) break;
            total = hSize + acc;
        }
        if (total >= n - 1) break;     // HUF_compressCTable_internal :1237
        cLit = total;
    } while (0);
    w.sync();
    ZB_PT(9);          // Huffman streams
    {   size_t const minGain = (n >> 6) + 2;
        if (cLit == 0 || isErr(cLit) || cLit >= n - minGain) return lit_raw(w, dst, cap, src, n); }
    if (cLit == 1) {
        // n >= 64 here, so the "single byte really is the whole literal run" check of :199-206 holds
        return lit_rle(w, dst, src, n);
    }
    if (w.lane == 0) {
        if (lhSize == 3) { u32 const lhc = 2 + ((u32)(!single) << 2) + ((u32)n << 4) + ((u32)cLit << 14); dst[0] = (u8)lhc; dst[1] = (u8)(lhc >> 8); dst[2] = (u8)(lhc >> 16); }
        else if (lhSize == 4) { u32 const lhc = 2 + (2 << 2) + ((u32)n << 4) + ((u32)cLit << 18); dst[0] = (u8)lhc; dst[1] = (u8)(lhc >> 8); dst[2] = (u8)(lhc >> 16); dst[3] = (u8)(lhc >> 24); }
        else { u32 const lhc = 2 + (3 << 2) + ((u32)n << 4) + ((u32)cLit << 22); dst[0] = (u8)lhc; dst[1] = (u8)(lhc >> 8); dst[2] = (u8)(lhc >> 16); dst[3] = (u8)(lhc >> 24); dst[4] = (u8)(cLit >> 10); }
    }
    w.sync();
    return lhSize + cLit;
}

// ------------------------------------------------------ sequences section
ZB_HD u32 ll_code(u32 ll) {   // ZSTD_LLcode, zstd_compress_internal.h:584-596
    if (ll > 63) return highbit32(ll) + 19;
    if (ll < 16) return ll;
    // 16..63 -> 16,16,17,17,18,18,19,19,20x4,21x4,22x8,23x8,24x16
    if (ll < 24) return 16 + ((ll - 16) >> 1);
    if (ll < 32) return 20 + ((ll - 24) >> 2);
    if (ll < 48) return 22 + ((ll - 32) >> 3);
    return 24;
}
ZB_HD u32 ml_code(u32 mlBase) {   // ZSTD_MLcode :601-613
    if (mlBase > 127) return highbit32(mlBase) + 36;
    if (mlBase < 32) return mlBase;
    // 32..127 -> 32,32,33,33,34,34,35,35,36x4,37x4,38x8,39x8,40x16,41x16,42x32
    if (mlBase < 40) return 32 + ((mlBase - 32) >> 1);
    if (mlBase < 48) return 36 + ((mlBase - 40) >> 2);
    if (mlBase < 64) return 38 + ((mlBase - 48) >> 3);
    if (mlBase < 96) return 40 + ((mlBase - 64) >> 4);
    return 42;
}
// ZSTD_selectEncodingType, first block, strategy < ZSTD_lazy (zstd_compress_sequences.c:156-204,232-234)
ZB_HD u32 select_encoding(size_t mostFrequent, size_t nbSeq, u32 defaultNormLog, bool defaultAllowed, u32 strategy) {
    if (mostFrequent == nbSeq) return (defaultAllowed && nbSeq <= 2) ? 0 : 1;
    if (defaultAllowed) {
        size_t const mult = 10 - strategy;
        size_t const dynamicFse_nbSeq_min = (((size_t)1 << defaultNormLog) * mult) >> 3;
        if ((nbSeq < dynamicFse_nbSeq_min) || (mostFrequent < (nbSeq >> (defaultNormLog - 1)))) return 0;
    }
    return 2;
}
// The same decision for strategy >= lazy (zstd_compress_sequences.c:205-231): estimated bit costs of the predefined
// table (ZSTD_crossEntropyCost :140-154) against a described one (ZSTD_NCountCost :71-79 + ZSTD_entropyCost :85-99);
// set_repeat cannot win in a first block.  One lane; S.norm and S.tableSymbol (512 B = FSE_NCOUNTBOUND) are scratch.
ZB_HDN u32 select_encoding_cost(EncShared& S, u32 max, size_t mostFrequent, size_t nbSeq, u32 FSELog, const i16* defaultNorm, u32 defaultNormLog, bool defaultAllowed) {
    if (mostFrequent == nbSeq) return (defaultAllowed && nbSeq <= 2) ? 0 : 1;
    size_t basicCost = (size_t)0 - 1;
    if (defaultAllowed) {
        u32 const shift = 8 - defaultNormLog; size_t cost = 0;
        for (u32 s = 0; s <= max; ++s) {
            u32 const normAcc = (defaultNorm[s] != -1) ? (u32)defaultNorm[s] : 1;
            cost += (size_t)S.count[s] * ZB_INVPROB[normAcc << shift];
        }
        basicCost = cost >> 8;
    }
    u32 const tableLog = fse_optimal_log(FSELog, nbSeq, max, 2);
    size_t r = fse_normalize(S.norm, tableLog, S.count, nbSeq, max, nbSeq >= 2048);
    if (!isErr(r)) r = fse_write_ncount(S.tableSymbol, sizeof(S.tableSymbol), S.norm, max, tableLog);
    u32 cost = 0;
    for (u32 s = 0; s <= max; ++s) {
        u32 norm256 = (u32)((256 * (u64)S.count[s]) / nbSeq);
        if (S.count[s] != 0 && norm256 == 0) norm256 = 1;
        cost += S.count[s] * ZB_INVPROB[norm256];
    }
    size_t const compressedCost = (r << 3) + (cost >> 8);
    return basicCost <= compressedCost ? 0 : 2;
}

// ZSTD_entropyCompressSeqStore_internal :2887-3003 on the block body; returns body size, 0 = emit raw block
template <class C>
ZB_HDN size_t entropy_compress(const C& w, EncShared& S, const EncWork& W, u8* dst, size_t cap, u32 nbSeq, size_t litSize, u32 strategy, bool disableLitCompression) {
    u8* op = dst; u8* const oend = dst + cap;
    ZB_PT_DECL
    {   bool const suspect = (nbSeq == 0) || (litSize / nbSeq >= 20);
        size_t const c = compress_literals(w, S, op, cap, W.lit, litSize, strategy, disableLitCompression, suspect);
        if (isErr(c)) return c;
        op += c; }
    ZB_PT(6);          // literals in total (= phases 7..9 + fallbacks)
    if ((oend - op) < 3 + 1) return ERR(E_dstSize_tooSmall);
    if (w.lane == 0) {
        if (nbSeq < 128) op[0] = (u8)nbSeq;
        else if (nbSeq < LONGNBSEQ) { op[0] = (u8)((nbSeq >> 8) + 0x80); op[1] = (u8)nbSeq; }
        else { op[0] = 0xFF; op[1] = (u8)(nbSeq - LONGNBSEQ); op[2] = (u8)((nbSeq - LONGNBSEQ) >> 8); }
    }
    op += (nbSeq < 128) ? 1 : (nbSeq < LONGNBSEQ) ? 2 : 3;
    if (nbSeq == 0) { w.sync(); return (size_t)(op - dst); }
    u8* const llc = W.codes; u8* const ofc = llc + MAX_SEQ; u8* const mlc = ofc + MAX_SEQ;
    for (u32 u = (u32)w.lane; u < nbSeq; u += C::W) {     // ZSTD_seqToCodes :2693-2719
        Seq const q = W.get(u);
        llc[u] = (u8)ll_code(q.ll);
        ofc[u] = (u8)highbit32(q.of);
        mlc[u] = (u8)ml_code(q.ml - MINMATCH);
    }
    w.sync();
    ZB_PT(2);          // seqToCodes
    u8* const seqHead = op++;
    size_t lastCountSize = 0; u32 types[3];
    // ZSTD_buildSequencesStatistics :2762-2880 : histogram on all lanes, table work on lane 0
    for (int t = 0; t < 3; t++) {
        const u8* const codes = t == 0 ? llc : t == 1 ? ofc : mlc;
        u32 max = t == 0 ? MaxLL : t == 1 ? MaxOff : MaxML;
        u32 const mf = hist_warp(w, S.count, &max, codes, nbSeq);
        bool const defaultAllowed = (t != 1) || (max <= DefaultMaxOff);
        u32 const dlog = t == 1 ? 5 : 6;
        u32 type;
        if (strategy < S_lazy) type = select_encoding(mf, nbSeq, dlog, defaultAllowed, strategy);
        else {
            type = 0;
            if (w.lane == 0) type = select_encoding_cost(S, max, mf, nbSeq, t == 1 ? OffFSELog : t == 0 ? LLFSELog : MLFSELog,
                                                         t == 0 ? ZB_T.LL_defaultNorm : t == 1 ? ZB_T.OF_defaultNorm : ZB_T.ML_defaultNorm, dlog, defaultAllowed);
            w.sync();
            type = w.bcast(type);
        }
        types[t] = type;
        size_t c = 0;
        if (w.lane == 0) {   // ZSTD_buildCTable, zstd_compress_sequences.c:242-288
            size_t const capLeft = (size_t)(oend - op);
            if (type == 1) { fse_build_ctable_rle(S.ctab(t), max); if (capLeft == 0) c = ERR(E_dstSize_tooSmall); else { op[0] = codes[0]; c = 1; } }
            else if (type == 0) {
                const i16* dn = t == 0 ? ZB_T.LL_defaultNorm : t == 1 ? ZB_T.OF_defaultNorm : ZB_T.ML_defaultNorm;
                u32 const dmax = t == 0 ? MaxLL : t == 1 ? DefaultMaxOff : MaxML;
                for (u32 s = 0; s <= dmax; s++) S.norm[s] = dn[s];
                fse_build_ctable(S.ctab(t), S.norm, dmax, dlog, S.cumul, S.tableSymbol);
                c = 0;
            } else {
                u32 const FSELog = t == 1 ? OffFSELog : LLFSELog;
                size_t nbSeq_1 = nbSeq; u32 const tableLog = fse_optimal_log(FSELog, nbSeq, max, 2);
                if (S.count[codes[nbSeq - 1]] > 1) { S.count[codes[nbSeq - 1]]--; nbSeq_1--; }
                size_t r = fse_normalize(S.norm, tableLog, S.count, nbSeq_1, max, nbSeq_1 >= 2048);
                if (!isErr(r)) r = fse_write_ncount(op, capLeft, S.norm, max, tableLog);
                if (!isErr(r)) fse_build_ctable(S.ctab(t), S.norm, max, tableLog, S.cumul, S.tableSymbol);
                c = r;
            }
        }
        w.sync();
        c = w.bcast(c);
        if (isErr(c)) return c;
        if (type == 2) lastCountSize = c;
        op += c;
    }
    // ZSTD_encodeSequences_body, zstd_compress_sequences.c:290-382, in two phases:
    //  1. the three FSE state chains (LL, OF, ML) are independent of each other: lanes 0..2 walk one each,
    //     last sequence to first, recording the bits every transition emits;
    //  2. all lanes pack the per-sequence bit groups (state bits OF,ML,LL then extra bits LL,ML,OF) at
    //     offsets from a prefix sum, the last lane appends the final states (ML,OF,LL) and the end mark.
    if (w.lane == 0) *seqHead = (u8)((types[0] << 6) + (types[1] << 4) + (types[2] << 2));
    ZB_PT(3);          // sequence statistics + tables
    size_t streamSize = 0;
    {
        u16* const stb = W.stbits;
        for (int t = w.lane; t < 3; t += C::W) {
            const u8* const codes = t == 0 ? llc : t == 1 ? ofc : mlc;
            const FseCT& ct = S.ctab(t);
            u16* const out = stb + (size_t)t * MAX_SEQ;
            u32 state = fse_init_state2(ct, codes[nbSeq - 1]);
            // Only state -> nbBits -> next state is serial.  The codes (global memory) are read four at a time one
            // group ahead and their transform entries (shared memory) are fetched before the group's chain starts, so
            // no memory access sits on the chain except the state-table lookup itself.
            u32 n = nbSeq - 1;                       // sequences n-1 .. 0 remain
            u32 ahead = n >= 4 ? load32(codes + (n - 4)) : 0;
            while (n >= 4) {
                u32 const cw = ahead;
                if (n >= 8) ahead = load32(codes + (n - 8));
                SymTT const t3 = ct.tt[cw >> 24], t2 = ct.tt[(cw >> 16) & 0xFF], t1 = ct.tt[(cw >> 8) & 0xFF], t0 = ct.tt[cw & 0xFF];
                u32 nb;
                nb = (state + t3.deltaNbBits) >> 16; out[n - 1] = (u16)((state & ((1u << nb) - 1)) | (nb << 12)); state = ct.stateTable[(int)(state >> nb) + t3.deltaFindState];
                nb = (state + t2.deltaNbBits) >> 16; out[n - 2] = (u16)((state & ((1u << nb) - 1)) | (nb << 12)); state = ct.stateTable[(int)(state >> nb) + t2.deltaFindState];
                nb = (state + t1.deltaNbBits) >> 16; out[n - 3] = (u16)((state & ((1u << nb) - 1)) | (nb << 12)); state = ct.stateTable[(int)(state >> nb) + t1.deltaFindState];
                nb = (state + t0.deltaNbBits) >> 16; out[n - 4] = (u16)((state & ((1u << nb) - 1)) | (nb << 12)); state = ct.stateTable[(int)(state >> nb) + t0.deltaFindState];
                n -= 4;
            }
            while (n-- > 0) {
                SymTT const tt = ct.tt[codes[n]];
                u32 const nb = (state + tt.deltaNbBits) >> 16;
                out[n] = (u16)((state & ((1u << nb) - 1)) | (nb << 12));
                state = ct.stateTable[(int)(state >> nb) + tt.deltaFindState];
            }
            S.tmp[t] = state;
        }
        w.sync();
        ZB_PT(4);      // FSE state chains
        // 2. bit packing, one row of C::W sequences at a time (lane = sequence, so every global access is coalesced; per-lane
        //    slices of the nine arrays used to thrash L1): bit offsets inside the row come from an exclusive scan, the
        //    fields are OR-ed into a shared-memory row buffer, whole bytes are flushed with coalesced stores and the
        //    partial last byte is carried into the next row.
        u32 mine = 0;
        for (u32 j = (u32)w.lane; j < nbSeq; j += C::W) {        // sizing pass
            u32 const n = nbSeq - 1 - j;
            mine += ZB_T.LL_bits[llc[n]] + ZB_T.ML_bits[mlc[n]] + ofc[n];
            if (j) mine += (stb[n] >> 12) + (stb[MAX_SEQ + n] >> 12) + (stb[2 * MAX_SEQ + n] >> 12);
        }
        u32 const seqBits = w.sum(mine);
        size_t const totalBits = (size_t)seqBits + S.ctab(0).tableLog + S.ctab(1).tableLog + S.ctab(2).tableLog + 1;
        size_t const capLeft = (size_t)(oend - op);
        if (capLeft <= 8 || (totalBits >> 3) >= capLeft - 8) return ERR(E_dstSize_tooSmall);
        streamSize = (totalBits + 7) >> 3;
        u32* const rowBuf = S.count;                     // the histogram is free now; a row needs at most (W * 90 + 7) bits
        const u8* const rowBytes = reinterpret_cast<const u8*>(rowBuf);
        u32 carryBits = 0, carryVal = 0; size_t outPos = 0;
        auto or_bits = [&](u32 pos, u32 v, u32 bits) {
            if (!bits) return;
            w.atomic_or32(&rowBuf[pos >> 5], v << (pos & 31));
            if ((pos & 31) + bits > 32) w.atomic_or32(&rowBuf[(pos >> 5) + 1], v >> (32 - (pos & 31)));
        };
        for (u32 base = 0; base < nbSeq; base += C::W) {
            u32 const j = base + (u32)w.lane; bool const valid = j < nbSeq;
            u32 const n = valid ? nbSeq - 1 - j : 0;
            u32 fo = 0, fm = 0, fl = 0, lbits = 0, mbits = 0, obits = 0, vl = 0, vm = 0, vo = 0;
            if (valid) {
                if (j) { fo = stb[MAX_SEQ + n]; fm = stb[2 * MAX_SEQ + n]; fl = stb[n]; }
                lbits = ZB_T.LL_bits[llc[n]]; mbits = ZB_T.ML_bits[mlc[n]]; obits = ofc[n];
                Seq const q = W.get(n);
                vl = q.ll & ((1u << lbits) - 1);
                vm = (q.ml - MINMATCH) & ((1u << mbits) - 1);
                vo = q.of & (obits >= 32 ? 0xFFFFFFFFu : ((1u << obits) - 1));
            }
            u32 const myBits = (fo >> 12) + (fm >> 12) + (fl >> 12) + lbits + mbits + obits;
            u32 const pre = w.exscan(myBits);
            u32 const rowBits = w.bcast(pre + myBits, C::W - 1) + carryBits;
            u32 const nWords = (rowBits + 31) >> 5;
            for (u32 i = (u32)w.lane; i <= nWords; i += C::W) rowBuf[i] = i ? 0 : carryVal;
            w.sync();
            if (valid) {
                u32 pos = pre + carryBits;
                or_bits(pos, fo & 0xFFF, fo >> 12); pos += fo >> 12;
                or_bits(pos, fm & 0xFFF, fm >> 12); pos += fm >> 12;
                or_bits(pos, fl & 0xFFF, fl >> 12); pos += fl >> 12;
                or_bits(pos, vl, lbits); pos += lbits;
                or_bits(pos, vm, mbits); pos += mbits;
                or_bits(pos, vo, obits);
            }
            w.sync();
            u32 const nBytes = rowBits >> 3;
            for (u32 i = (u32)w.lane; i < nBytes; i += C::W) op[outPos + i] = rowBytes[i];
            carryBits = rowBits & 7;
            carryVal = carryBits ? (u32)rowBytes[nBytes] & ((1u << carryBits) - 1) : 0;
            outPos += nBytes;
            w.sync();
        }
        if (w.lane == 0) {      // final states (ML, OF, LL), the end mark, and whatever the last row left over
            u64 acc = carryVal; u32 nb = carryBits;
            acc |= (u64)(S.tmp[2] & ((1u << S.ctab(2).tableLog) - 1)) << nb; nb += S.ctab(2).tableLog;
            acc |= (u64)(S.tmp[1] & ((1u << S.ctab(1).tableLog) - 1)) << nb; nb += S.ctab(1).tableLog;
            acc |= (u64)(S.tmp[0] & ((1u << S.ctab(0).tableLog) - 1)) << nb; nb += S.ctab(0).tableLog;
            acc |= (u64)1 << nb; nb += 1;
            for (u32 i = 0; i * 8 < nb; i++) op[outPos + i] = (u8)(acc >> (8 * i));
        }
        w.sync();
    }
    ZB_PT(5);          // sequence bit packing
    op += streamSize;
    if (lastCountSize && (lastCountSize + streamSize) < 4) return 0;    // :2992-2998
    return (size_t)(op - dst);
}

// ZSTD_compressBlock_fast_noDict_generic, N/compress/zstd_fast.c:190-423, fresh frame, serial.
// The reference software-pipelines positions ip0..ip3; the order of table writes and reads
// is observable in the output, so it is kept.
ZB_HD bool match4(const u8* cur, const u8* base, u32 idx) { return idx >= 2 && load32(cur) == load32(base + idx); }
ZB_HDN u32 parse_fast(const EncWork& W, const u8* src, size_t srcSize, u32 hlog, u32 mls, u32 targetLength, u32* lastLL) {
    u32* const hashTable = W.hashLong;
    u32 const stepSize = targetLength + !targetLength + 1;
    const u8* const base = src - 2;
    const u8* const prefixStart = src;
    const u8* const iend = src + srcSize;
    const u8* const ilimit = iend - 8;
    const u8* anchor = src; const u8* ip0 = src + 1; const u8* ip1; const u8* ip2; const u8* ip3;
    u32 current0 = 0, rep1 = 1, rep2 = 4, nbSeq = 0;
    {   u32 const maxRep = 1;
        if (rep2 > maxRep) rep2 = 0;
        if (rep1 > maxRep) rep1 = 0; }
    for (;;) {   // _start
        u32 step = stepSize; const u8* nextStep = ip0 + 128;
        u32 hash0, hash1, matchIdx, mLength = 0, offcode = 0; const u8* match0 = nullptr; int kind = 0;   // 1 = repcode, 2 = hash match
        ip1 = ip0 + 1; ip2 = ip0 + step; ip3 = ip2 + 1;
        if (ip3 >= ilimit) break;
        hash0 = hash_ptr(ip0, hlog, mls); hash1 = hash_ptr(ip1, hlog, mls);
        matchIdx = hashTable[hash0];
        do {
            u32 const rval = load32(ip2 - rep1);
            current0 = (u32)(ip0 - base);
            hashTable[hash0] = current0;
            if ((load32(ip2) == rval) & (rep1 > 0)) {
                ip0 = ip2; match0 = ip0 - rep1;
                mLength = ip0[-1] == match0[-1];
                ip0 -= mLength; match0 -= mLength;
                offcode = 1; mLength += 4;
                hashTable[hash1] = (u32)(ip1 - base);
                kind = 1; break;
            }
            if (match4(ip0, base, matchIdx)) { hashTable[hash1] = (u32)(ip1 - base); kind = 2; break; }
            matchIdx = hashTable[hash1];
            hash0 = hash1; hash1 = hash_ptr(ip2, hlog, mls);
            ip0 = ip1; ip1 = ip2; ip2 = ip3;
            current0 = (u32)(ip0 - base);
            hashTable[hash0] = current0;
            if (match4(ip0, base, matchIdx)) { if (step <= 4) hashTable[hash1] = (u32)(ip1 - base); kind = 2; break; }
            matchIdx = hashTable[hash1];
            hash0 = hash1; hash1 = hash_ptr(ip2, hlog, mls);
            ip0 = ip1; ip1 = ip2; ip2 = ip0 + step; ip3 = ip1 + step;
            if (ip2 >= nextStep) { step++; nextStep += 128; }
        } while (ip3 < ilimit);
        if (kind == 0) break;
        if (kind == 2) {
            match0 = base + matchIdx;
            rep2 = rep1; rep1 = (u32)(ip0 - match0);
            offcode = rep1 + 3; mLength = 4;
            while (((ip0 > anchor) & (match0 > prefixStart)) && (ip0[-1] == match0[-1])) { ip0--; match0--; mLength++; }
        }
        mLength += count_match(ip0 + mLength, match0 + mLength, iend);
        W.put(nbSeq, (u32)(ip0 - anchor), offcode, mLength); nbSeq++;
        ip0 += mLength; anchor = ip0;
        if (ip0 <= ilimit) {
            hashTable[hash_ptr(base + current0 + 2, hlog, mls)] = current0 + 2;
            hashTable[hash_ptr(ip0 - 2, hlog, mls)] = (u32)(ip0 - 2 - base);
            if (rep2 > 0) {
                while ((ip0 <= ilimit) && (load32(ip0) == load32(ip0 - rep2))) {
                    u32 const rLength = count_match(ip0 + 4, ip0 + 4 - rep2, iend) + 4;
                    { u32 const t = rep2; rep2 = rep1; rep1 = t; }
                    hashTable[hash_ptr(ip0, hlog, mls)] = (u32)(ip0 - base);
                    ip0 += rLength;
                    W.put(nbSeq, 0, 1, rLength); nbSeq++;
                    anchor = ip0;
                }
            }
        }
    }
    *lastLL = (u32)(iend - anchor);
    return nbSeq;
}

// Cooperative version of parse_fast (ZSTD_compressBlock_fast_noDict_generic, zstd_fast.c:190-423) for levels 1, 2 and
// the negative levels.  The reference visits positions in pairs: iteration i hashes a_i and a_i + 1 and tests the
// repcode at r_i = a_{i+1} (the next pair), in the order [rep @ r_i] -> [hash @ a_i] -> [hash @ a_i + 1]; every visited
// position is written to the table before the next one is read.  Here lane 2i / 2i+1 take a_i / a_i + 1 of up to 16
// consecutive iterations: table reads are forwarded between lanes exactly like in parse_dfast_warp, the first event
// in the reference's order ends the batch, and only what the serial code would have written is committed.
// Iteration state (a, r, s, nextStep): rep test at r, then a' = r, r' = a' + s, and s grows when r' reaches nextStep
// (the reference computes ip2 before it bumps `step`, hence the explicit r).  Cells carry a 14-bit fingerprint.
template <class C>
ZB_HDN u32 parse_fast_warp(const C& w, const EncWork& W, const u8* src, size_t srcSize, u32 hlog, u32 mls, u32 targetLength, u32* lastLL) {
    u32* const T = W.hashLong;
    u32 const stepSize = targetLength + !targetLength + 1;
    int const n = (int)srcSize, ilimit = n - 8;
    int ip0 = 1, anchor = 0;
    u32 rep1 = 1, rep2 = 0, nbSeq = 0;          // {1,4,8} clipped by maxRep = 1 at position 1
    u32 const lane = (u32)w.lane;
    int const it = (int)(lane >> 1); bool const odd = (lane & 1) != 0;
    u32 est4 = 4 * 3;
    bool done = false;
    while (!done) {   // _start: one iteration per stored match
        if (ip0 + (int)stepSize + 1 >= ilimit) break;
        int a = ip0, r = ip0 + (int)stepSize, nextStep = ip0 + 128; u32 s = stepSize;      // state of the first iteration
        u32 nIt = 1;
        {   u32 const want = (est4 + 7) / 8;
            while (nIt < want && 2 * nIt < (u32)C::W) nIt *= 2; }
        u32 runIt = 0;
        int evKey = -1, e = -1;
        // per-lane values of the deciding batch
        int ai = 0, ri = 0; u32 si = 0; int nsi = 0; u64 d = 0; u32 h = 0, idx = 0; int p = 0;
        for (;;) {   // batches of nIt iterations
            // my iteration's start state (ai, ri, si, nsi) and its end state (ae, re, se, nse)
            ai = a; ri = r; si = s; nsi = nextStep;
            if (r + (int)(C::W / 2 + 1) * (int)s < nextStep) { if (it > 0) { ai = r + (it - 1) * (int)s; ri = r + it * (int)s; } }
            else for (int j = 0; j < it; j++) { ai = ri; ri = ai + (int)si; if (ri >= nsi) { si++; nsi += 128; } }
            int ae = ri, re = ae + (int)si; u32 se = si; int nse = nsi;
            if (re >= nse) { se++; nse += 128; }
            bool const valid = (u32)it < nIt && ri + 1 < ilimit;        // monotone in it
            bool const active = valid && lane < (u32)C::W;
            p = ai + (odd ? 1 : 0);
            d = active ? load64(src + p) : 0;
            h = hashSv(d, hlog, mls);
            u32 const myTag = tag4((u32)d);
            u32 const tv = active ? ld_probe32(T + h) : 0;
            u32 const mH = w.match_any(active ? h : (0x80000000u | lane));
            u32 const lowH = mH & ((1u << lane) - 1);
            int const pLow = w.shfl(p, lowH ? (int)highbit32(lowH) : (int)lane);
            idx = lowH ? (u32)pLow + 2 : (tv & CELL_IDX_MASK);
            bool const plaus = idx >= 2 && (lowH || (tv >> 18) == myTag);
            bool const hashOk = active && plaus && (load32(src + (idx - 2)) == (u32)d);
            bool const repOk = active && !odd && rep1 > 0 && (load32(src + ri) == load32(src + ri - (int)rep1));
            u32 const repMask = w.ballot(repOk), hashMask = w.ballot(hashOk);
            u32 const nValid = popc32(w.ballot(active && !odd));
            int const keyR = repMask ? 3 * (int)(ctz32(repMask) >> 1) : 0x7FFFFFFF;
            int const lh = hashMask ? (int)ctz32(hashMask) : 0;
            int const keyH = hashMask ? 3 * (lh >> 1) + 1 + (lh & 1) : 0x7FFFFFFF;
            evKey = keyR < keyH ? keyR : keyH;
            if (evKey == 0x7FFFFFFF) evKey = -1;
            e = evKey >= 0 ? evKey / 3 : -1;
            // commits: every active lane up to 2e+1 (all of them without event); per cell only the last writer
            int const lastLane = evKey >= 0 ? 2 * e + 1 : 2 * (int)nValid - 1;
            if (active && (int)lane <= lastLane) {
                u32 const later = ((lastLane >= 31) ? 0xFFFFFFFFu : ((2u << lastLane) - 1)) & ~((2u << lane) - 1);
                if (!(mH & later)) T[h] = cell((u32)p + 2, myTag);
            }
            w.sync();
            runIt += evKey >= 0 ? (u32)e + 1 : nValid;
            if (evKey >= 0) break;
            if (nValid < nIt) { done = true; break; }          // ran into ilimit: the reference leaves the search loop for good
            {   int const L = 2 * ((int)nValid - 1);
                a = w.shfl(ae, L); r = w.shfl(re, L); s = w.shfl(se, L); nextStep = w.shfl(nse, L); }
            if (r + 1 >= ilimit) { done = true; break; }
            nIt = 2 * nIt * 2 <= (u32)C::W ? nIt * 2 : (u32)C::W / 2;
        }
        if (done || evKey < 0) break;
        est4 = (3 * est4 + 4 * 2 * (runIt < 32 ? runIt : 32)) / 4;
        // ---- event in iteration e
        int const kindE = evKey - 3 * e;                      // 0 rep @ r_e, 1 hash @ a_e, 2 hash @ a_e + 1
        int const aE = w.shfl(ai, 2 * e), rE = w.shfl(ri, 2 * e); u32 const sE = w.shfl(si, 2 * e);
        u32 mLength; int mpos, cur;
        if (kindE == 2 && sE <= 4) {                          // :"if (step <= 4) hashTable[hash1] = ip1" with ip1 == r_e
            if (lane == 0) { u64 const dr = load64(src + rE); T[hashSv(dr, hlog, mls)] = cell((u32)rE + 2, tag4((u32)dr)); }
        }
        if (kindE == 0) {
            cur = aE; ip0 = rE; mpos = ip0 - (int)rep1;
            u32 const back = (src[ip0 - 1] == src[mpos - 1]) ? 1u : 0u;
            ip0 -= (int)back; mpos -= (int)back;
            mLength = 4 + back;
            mLength += wcount(w, src, (u32)n, (u32)ip0 + mLength, (u32)mpos + mLength);
            if (lane == 0) { W.put(nbSeq, (u32)(ip0 - anchor), 1, mLength); }
        } else {
            int const le = 2 * e + (kindE == 2 ? 1 : 0);
            ip0 = aE + (kindE == 2 ? 1 : 0); cur = ip0;
            mpos = (int)w.shfl(idx, le) - 2;
            rep2 = rep1; rep1 = (u32)(ip0 - mpos);
            u32 const maxBack = (u32)(ip0 - anchor) < (u32)mpos ? (u32)(ip0 - anchor) : (u32)mpos;
            u32 const back = maxBack ? wcatchup(w, src, (u32)ip0, (u32)mpos, maxBack) : 0;
            u32 const fwd = wcount(w, src, (u32)n, (u32)ip0 + 4, (u32)mpos + 4);
            ip0 -= (int)back; mLength = 4 + back + fwd;
            if (lane == 0) { W.put(nbSeq, (u32)(ip0 - anchor), rep1 + 3, mLength); }
        }
        nbSeq++;
        ip0 += (int)mLength; anchor = ip0;
        w.sync();
        if (ip0 <= ilimit) {
            if (lane == 0) {   // :"Fill table and check for immediate repcode"
                u64 const dA = load64(src + cur + 2), dB = load64(src + ip0 - 2);
                T[hashSv(dA, hlog, mls)] = cell((u32)cur + 2 + 2, tag4((u32)dA));
                T[hashSv(dB, hlog, mls)] = cell((u32)ip0 - 2 + 2, tag4((u32)dB));
            }
            w.sync();
            if (rep2 > 0) {
                while ((ip0 <= ilimit) && (load32(src + ip0) == load32(src + ip0 - (int)rep2))) {
                    u32 const rLength = wcount(w, src, (u32)n, (u32)ip0 + 4, (u32)ip0 + 4 - rep2) + 4;
                    { u32 const t = rep2; rep2 = rep1; rep1 = t; }
                    if (lane == 0) {
                        u64 const d0 = load64(src + ip0);
                        T[hashSv(d0, hlog, mls)] = cell((u32)ip0 + 2, tag4((u32)d0));
                        W.put(nbSeq, 0, 1, rLength);
                    }
                    nbSeq++; ip0 += (int)rLength; anchor = ip0;
                    w.sync();
                }
            }
        }
    }
    w.sync();
    *lastLL = (u32)(n - anchor);
    return nbSeq;
}

// ZSTD_compressBlock_lazy_generic (N/compress/zstd_lazy.c:1516-1779; depth 0 greedy, 1 lazy, 2 lazy2) with the
// row-based match finder (ZSTD_RowFindBestMatch :1141-1283, ZSTD_row_update_internal :885-943, hash cache :837-878,
// ZSTD_row_nextIndex :798-803, match mask :1061-1121), fresh frame, no dictionary.  Serial: call from one lane.
// hashTable = W.hashLong (1 << hashLog cells), tag rows = the bytes of W.hashSmall; index = position + 2.
// The hash salt is 0 (it only permutes rows and tags, the sequences do not depend on it).
struct RowState {
    u32* hashTable; u8* tagTable; const u8* base;
    u32 hashCache[8];
    u32 hc;                     // full-warp parsers: lane k (k < 8) holds hashCache[k] in this register instead (a shuffle reads it)
    u32 rowHashLog, rowLog, searchLog, mls, nextToUpdate; bool lazySkipping;
    u32 finder;                 // 0 = hash chain (window <= 2^14), 1 = row based, 2 = binary tree (btlazy2)
    u32* chainTable; u32 hashLog, chainLog;
};
ZB_HD u32 row_hash(const u8* p, u32 hBits, u32 mls) {
    switch (mls) {
    default:
    case 4: return (load32(p) * 2654435761U) >> (32 - hBits);
    case 5: return (u32)(((load64(p) << 24) * 889523592379ULL) >> (64 - hBits));
    case 6: return (u32)(((load64(p) << 16) * 227718039650203ULL) >> (64 - hBits));
    }
}
ZB_HD u32 row_next_index(u8* tagRow, u32 rowMask) {
    u32 next = ((u32)*tagRow - 1) & rowMask;
    next += (next == 0) ? rowMask : 0;
    *tagRow = (u8)next;
    return next;
}
// The hash cache is the reference's latency trick (ZSTD_row_prefetch :816-829): the row of position idx + 8 is
// requested while position idx is searched.  Same here, towards L2: tag row (<= 64 B) and index row (<= 256 B).
ZB_HD void row_prefetch(const RowState& ms, u32 hash) {
    u32 const relRow = (hash >> 8) << ms.rowLog;
    prefetch_l2(ms.tagTable + relRow);            // (towards L1 instead: no gain at level 9, 3 % slower at level 5)
    prefetch_l2(ms.hashTable + relRow);
    if (ms.rowLog == 6) prefetch_l2(ms.hashTable + relRow + 32);
}
ZB_HD void row_fill_cache(RowState& ms, u32 idx, const u8* iLimit) {
    u32 const maxElems = (ms.base + idx) > iLimit ? 0 : (u32)(iLimit - (ms.base + idx) + 1);
    u32 const lim = idx + (8 < maxElems ? 8 : maxElems);
    for (; idx < lim; ++idx) { u32 const h = row_hash(ms.base + idx, ms.rowHashLog + 8, ms.mls); row_prefetch(ms, h); ms.hashCache[idx & 7] = h; }
}
ZB_HD u32 row_next_cached(RowState& ms, u32 idx) {
    u32 const newHash = row_hash(ms.base + idx + 8, ms.rowHashLog + 8, ms.mls);
    row_prefetch(ms, newHash);
    u32 const hash = ms.hashCache[idx & 7];
    ms.hashCache[idx & 7] = newHash;
    return hash;
}
ZB_HD void row_update_impl(RowState& ms, u32 idx, u32 end) {
    u32 const rowMask = (1u << ms.rowLog) - 1;
    for (; idx < end; ++idx) {
        u32 const hash = row_next_cached(ms, idx);
        u32 const relRow = (hash >> 8) << ms.rowLog;
        u8* const tagRow = ms.tagTable + relRow;
        u32 const pos = row_next_index(tagRow, rowMask);
        tagRow[pos] = (u8)hash;
        ms.hashTable[relRow + pos] = idx;
    }
}
ZB_HD void row_update(RowState& ms, const u8* ip) {
    u32 idx = ms.nextToUpdate;
    u32 const target = (u32)(ip - ms.base);
    if (target - idx > 384) {      // kSkipThreshold: only the first 96 and the last 32 positions of a long match are inserted
        row_update_impl(ms, idx, idx + 96);
        idx = target - 32;
        row_fill_cache(ms, idx, ip + 1);
    }
    row_update_impl(ms, idx, target);
    ms.nextToUpdate = target;
}
ZB_HDN size_t row_find_best(RowState& ms, const u8* ip, const u8* iLimit, size_t* offBasePtr) {
    u32 const curr = (u32)(ip - ms.base);
    u32 const lowLimit = 2;
    u32 const rowEntries = 1u << ms.rowLog, rowMask = rowEntries - 1;
    u32 nbAttempts = 1u << (ms.searchLog < ms.rowLog ? ms.searchLog : ms.rowLog);
    size_t ml = 4 - 1;
    u32 hash;
    if (!ms.lazySkipping) { row_update(ms, ip); hash = row_next_cached(ms, curr); }
    else { hash = row_hash(ip, ms.rowHashLog + 8, ms.mls); ms.nextToUpdate = curr; }
    u32 const relRow = (hash >> 8) << ms.rowLog;
    u32 const tag = hash & 0xFF;
    u32* const row = ms.hashTable + relRow;
    u8* const tagRow = ms.tagTable + relRow;
    u32 const head = *tagRow & rowMask;
    u32 matchBuffer[64]; u32 numMatches = 0;
    // the reference walks the tag-match mask rotated by head from bit 0: entries head, head+1, ... (mod rowEntries)
    for (u32 k = 0; k < rowEntries && nbAttempts > 0; k++) {
        u32 const matchPos = (head + k) & rowMask;
        if (tagRow[matchPos] != (u8)tag) continue;
        u32 const matchIndex = row[matchPos];
        if (matchPos == 0) continue;
        if (matchIndex < lowLimit) break;
        matchBuffer[numMatches++] = matchIndex;
        --nbAttempts;
    }
    {   u32 const pos = row_next_index(tagRow, rowMask);
        tagRow[pos] = (u8)tag;
        row[pos] = ms.nextToUpdate++; }
    for (u32 m = 0; m < numMatches; ++m) {
        const u8* const match = ms.base + matchBuffer[m];
        size_t currentMl = 0;
        if (load32(match + ml - 3) == load32(ip + ml - 3)) currentMl = count_match(ip, match, iLimit);
        if (currentMl > ml) {
            ml = currentMl;
            *offBasePtr = (size_t)(curr - matchBuffer[m]) + 3;
            if (ip + currentMl == iLimit) break;
        }
    }
    return ml;
}
// ZSTD_HcFindBestMatch :667-733 with ZSTD_insertAndFindFirstIndex_internal :632-657 (noDict): hashTable = W.hashLong,
// chainTable = W.hashSmall (1 << chainLog cells).
ZB_HDN size_t hc_find_best(RowState& ms, const u8* ip, const u8* iLimit, size_t* offBasePtr) {
    u32 const chainSize = 1u << ms.chainLog, chainMask = chainSize - 1;
    u32 const curr = (u32)(ip - ms.base);
    u32 const lowLimit = 2;
    u32 const minChain = curr > chainSize ? curr - chainSize : 0;
    u32 nbAttempts = 1u << ms.searchLog;
    size_t ml = 4 - 1;
    u32 matchIndex;
    {   u32 idx = ms.nextToUpdate;
        while (idx < curr) {
            u32 const h = row_hash(ms.base + idx, ms.hashLog, ms.mls);
            ms.chainTable[idx & chainMask] = ms.hashTable[h];
            ms.hashTable[h] = idx;
            idx++;
            if (ms.lazySkipping) break;
        }
        ms.nextToUpdate = curr;
        matchIndex = ms.hashTable[row_hash(ip, ms.hashLog, ms.mls)]; }
    for (; (matchIndex >= lowLimit) && (nbAttempts > 0); nbAttempts--) {
        const u8* const match = ms.base + matchIndex;
        size_t currentMl = 0;
        if (load32(match + ml - 3) == load32(ip + ml - 3)) currentMl = count_match(ip, match, iLimit);
        if (currentMl > ml) {
            ml = currentMl;
            *offBasePtr = (size_t)(curr - matchIndex) + 3;
            if (ip + currentMl == iLimit) break;
        }
        if (matchIndex <= minChain) break;
        matchIndex = ms.chainTable[matchIndex & chainMask];
    }
    return ml;
}
// Binary tree of the "dual unsorted" kind: ZSTD_BtFindBestMatch :399-408, ZSTD_updateDUBT :29-65, ZSTD_insertDUBT1 :74-163,
// ZSTD_DUBT_findBestMatch :243-395 (noDict).  bt = W.hashSmall as pairs {smaller, larger}, btLog = chainLog - 1.
ZB_HDN void dubt_insert1(RowState& ms, u32 curr, const u8* iend, u32 nbCompares, u32 btLow) {
    u32* const bt = ms.chainTable;
    u32 const btMask = (1u << (ms.chainLog - 1)) - 1;
    size_t commonLengthSmaller = 0, commonLengthLarger = 0;
    const u8* const ip = ms.base + curr;
    u32* smallerPtr = bt + 2 * (curr & btMask);
    u32* largerPtr = smallerPtr + 1;
    u32 matchIndex = *smallerPtr;
    u32 dummy32;
    for (; nbCompares && (matchIndex > 2); --nbCompares) {
        u32* const nextPtr = bt + 2 * (matchIndex & btMask);
        size_t matchLength = commonLengthSmaller < commonLengthLarger ? commonLengthSmaller : commonLengthLarger;
        const u8* const match = ms.base + matchIndex;
        matchLength += count_match(ip + matchLength, match + matchLength, iend);
        if (ip + matchLength == iend) break;
        if (match[matchLength] < ip[matchLength]) {
            *smallerPtr = matchIndex; commonLengthSmaller = matchLength;
            if (matchIndex <= btLow) { smallerPtr = &dummy32; break; }
            smallerPtr = nextPtr + 1; matchIndex = nextPtr[1];
        } else {
            *largerPtr = matchIndex; commonLengthLarger = matchLength;
            if (matchIndex <= btLow) { largerPtr = &dummy32; break; }
            largerPtr = nextPtr; matchIndex = nextPtr[0];
        }
    }
    *smallerPtr = *largerPtr = 0;
}
ZB_HDN size_t bt_find_best(RowState& ms, const u8* ip, const u8* iend, size_t* offBasePtr) {
    u32* const bt = ms.chainTable;
    u32 const btMask = (1u << (ms.chainLog - 1)) - 1;
    u32 const curr = (u32)(ip - ms.base);
    u32 const windowLow = 2;
    u32 const btLow = (btMask >= curr) ? 0 : curr - btMask;
    u32 const unsortLimit = btLow > windowLow ? btLow : windowLow;
    u32 nbCompares = 1u << ms.searchLog, nbCandidates = nbCompares, previousCandidate = 0;
    if (ip < ms.base + ms.nextToUpdate) return 0;      // skipped area
    for (u32 idx = ms.nextToUpdate; idx < curr; idx++) {      // ZSTD_updateDUBT
        u32 const hh = row_hash(ms.base + idx, ms.hashLog, ms.mls);
        u32* const nc = bt + 2 * (idx & btMask);
        nc[0] = ms.hashTable[hh]; nc[1] = 1;          // ZSTD_DUBT_UNSORTED_MARK
        ms.hashTable[hh] = idx;
    }
    ms.nextToUpdate = curr;
    u32 const h = row_hash(ip, ms.hashLog, ms.mls);
    u32 matchIndex = ms.hashTable[h];
    u32* nextCandidate = bt + 2 * (matchIndex & btMask); u32* unsortedMark = nextCandidate + 1;
    while ((matchIndex > unsortLimit) && (*unsortedMark == 1) && (nbCandidates > 1)) {
        *unsortedMark = previousCandidate;
        previousCandidate = matchIndex;
        matchIndex = *nextCandidate;
        nextCandidate = bt + 2 * (matchIndex & btMask); unsortedMark = nextCandidate + 1;
        nbCandidates--;
    }
    if ((matchIndex > unsortLimit) && (*unsortedMark == 1)) *nextCandidate = *unsortedMark = 0;
    matchIndex = previousCandidate;
    while (matchIndex) {
        u32 const nextCandidateIdx = bt[2 * (matchIndex & btMask) + 1];
        dubt_insert1(ms, matchIndex, iend, nbCandidates, unsortLimit);
        matchIndex = nextCandidateIdx;
        nbCandidates++;
    }
    size_t commonLengthSmaller = 0, commonLengthLarger = 0, bestLength = 0;
    u32* smallerPtr = bt + 2 * (curr & btMask);
    u32* largerPtr = smallerPtr + 1;
    u32 matchEndIdx = curr + 8 + 1;
    u32 dummy32;
    matchIndex = ms.hashTable[h];
    ms.hashTable[h] = curr;
    for (; nbCompares && (matchIndex > windowLow); --nbCompares) {
        u32* const nextPtr = bt + 2 * (matchIndex & btMask);
        size_t matchLength = commonLengthSmaller < commonLengthLarger ? commonLengthSmaller : commonLengthLarger;
        const u8* const match = ms.base + matchIndex;
        matchLength += count_match(ip + matchLength, match + matchLength, iend);
        if (matchLength > bestLength) {
            if (matchLength > matchEndIdx - matchIndex) matchEndIdx = matchIndex + (u32)matchLength;
            if ((4 * (int)(matchLength - bestLength)) > (int)(highbit32(curr - matchIndex + 1) - highbit32((u32)*offBasePtr))) {
                bestLength = matchLength; *offBasePtr = (size_t)(curr - matchIndex) + 3; }
            if (ip + matchLength == iend) break;
        }
        if (match[matchLength] < ip[matchLength]) {
            *smallerPtr = matchIndex; commonLengthSmaller = matchLength;
            if (matchIndex <= btLow) { smallerPtr = &dummy32; break; }
            smallerPtr = nextPtr + 1; matchIndex = nextPtr[1];
        } else {
            *largerPtr = matchIndex; commonLengthLarger = matchLength;
            if (matchIndex <= btLow) { largerPtr = &dummy32; break; }
            largerPtr = nextPtr; matchIndex = nextPtr[0];
        }
    }
    *smallerPtr = *largerPtr = 0;
    ms.nextToUpdate = matchEndIdx - 8;
    return bestLength;
}
ZB_HD size_t lazy_find_best(RowState& ms, const u8* ip, const u8* iLimit, size_t* offBasePtr) {
    if (ms.finder == 2) return bt_find_best(ms, ip, iLimit, offBasePtr);
    return ms.finder == 1 ? row_find_best(ms, ip, iLimit, offBasePtr) : hc_find_best(ms, ip, iLimit, offBasePtr);
}
ZB_HDN u32 parse_lazy(const EncWork& W, const u8* src, size_t srcSize, u32 hashLog, u32 chainLog, u32 searchLog, u32 minMatch, u32 depth, u32 finder, u32* lastLL) {
    bool const useRow = finder == 1;
    const u8* const istart = src;
    const u8* ip = istart;
    const u8* anchor = istart;
    const u8* const iend = istart + srcSize;
    const u8* const ilimit = useRow ? iend - 8 - 8 : iend - 8;
    const u8* const prefixLowest = src;
    u32 offset_1 = 1, offset_2 = 4, nbSeq = 0;
    RowState ms;
    ms.finder = finder; ms.chainTable = W.hashSmall; ms.hashLog = hashLog; ms.chainLog = chainLog;
    ms.hashTable = W.hashLong; ms.tagTable = reinterpret_cast<u8*>(W.hashSmall); ms.base = src - 2;
    ms.mls = minMatch < 4 ? 4 : minMatch > 6 ? 6 : minMatch;
    ms.rowLog = searchLog < 4 ? 4 : searchLog > 6 ? 6 : searchLog;
    ms.searchLog = searchLog; ms.rowHashLog = hashLog - ms.rowLog;
    ms.nextToUpdate = 2; ms.lazySkipping = false;
    ip += 1;
    {   u32 const maxRep = (u32)(ip - prefixLowest);
        if (offset_2 > maxRep) offset_2 = 0;
        if (offset_1 > maxRep) offset_1 = 0; }
    if (useRow) row_fill_cache(ms, ms.nextToUpdate, ilimit);
    while (ip < ilimit) {
        size_t matchLength = 0;
        size_t offBase = 1;
        const u8* start = ip + 1;
        bool store = false;
        if ((offset_1 > 0) && (load32(ip + 1 - offset_1) == load32(ip + 1))) {
            matchLength = count_match(ip + 1 + 4, ip + 1 + 4 - offset_1, iend) + 4;
            if (depth == 0) store = true;
        }
        if (!store) {
            {   size_t offbaseFound = 999999999;
                size_t const ml2 = lazy_find_best(ms, ip, iend, &offbaseFound);
                if (ml2 > matchLength) { matchLength = ml2; start = ip; offBase = offbaseFound; } }
            if (matchLength < 4) {
                size_t const step = ((size_t)(ip - anchor) >> 8) + 1;      // kSearchStrength
                ip += step;
                ms.lazySkipping = step > 8;                                // kLazySkippingStep
                continue;
            }
            if (depth >= 1)
            while (ip < ilimit) {
                ip++;
                if ((offBase) && ((offset_1 > 0) && (load32(ip) == load32(ip - offset_1)))) {
                    size_t const mlRep = count_match(ip + 4, ip + 4 - offset_1, iend) + 4;
                    int const gain2 = (int)(mlRep * 3);
                    int const gain1 = (int)(matchLength * 3 - highbit32((u32)offBase) + 1);
                    if ((mlRep >= 4) && (gain2 > gain1)) { matchLength = mlRep; offBase = 1; start = ip; }
                }
                {   size_t ofbCandidate = 999999999;
                    size_t const ml2 = lazy_find_best(ms, ip, iend, &ofbCandidate);
                    int const gain2 = (int)(ml2 * 4 - highbit32((u32)ofbCandidate));
                    int const gain1 = (int)(matchLength * 4 - highbit32((u32)offBase) + 4);
                    if ((ml2 >= 4) && (gain2 > gain1)) { matchLength = ml2; offBase = ofbCandidate; start = ip; continue; } }
                if ((depth == 2) && (ip < ilimit)) {
                    ip++;
                    if ((offBase) && ((offset_1 > 0) && (load32(ip) == load32(ip - offset_1)))) {
                        size_t const mlRep = count_match(ip + 4, ip + 4 - offset_1, iend) + 4;
                        int const gain2 = (int)(mlRep * 4);
                        int const gain1 = (int)(matchLength * 4 - highbit32((u32)offBase) + 1);
                        if ((mlRep >= 4) && (gain2 > gain1)) { matchLength = mlRep; offBase = 1; start = ip; }
                    }
                    {   size_t ofbCandidate = 999999999;
                        size_t const ml2 = lazy_find_best(ms, ip, iend, &ofbCandidate);
                        int const gain2 = (int)(ml2 * 4 - highbit32((u32)ofbCandidate));
                        int const gain1 = (int)(matchLength * 4 - highbit32((u32)offBase) + 7);
                        if ((ml2 >= 4) && (gain2 > gain1)) { matchLength = ml2; offBase = ofbCandidate; start = ip; continue; } }
                }
                break;
            }
            if (offBase > 3) {   // catch up
                size_t const off = offBase - 3;
                while (((start > anchor) && (start - off > prefixLowest)) && (start[-1] == (start - off)[-1])) { start--; matchLength++; }
                offset_2 = offset_1; offset_1 = (u32)off;
            }
        }
        W.put(nbSeq, (u32)(start - anchor), (u32)offBase, (u32)matchLength); nbSeq++;
        anchor = ip = start + matchLength;
        if (ms.lazySkipping) { if (useRow) row_fill_cache(ms, ms.nextToUpdate, ilimit); ms.lazySkipping = false; }
        while (((ip <= ilimit) && (offset_2 > 0)) && (load32(ip) == load32(ip - offset_2))) {
            matchLength = count_match(ip + 4, ip + 4 - offset_2, iend) + 4;
            u32 const tmp = offset_2; offset_2 = offset_1; offset_1 = tmp;
            W.put(nbSeq, 0, 1, (u32)matchLength); nbSeq++;
            ip += matchLength; anchor = ip;
        }
    }
    *lastLL = (u32)(iend - anchor);
    return nbSeq;
}

// ---- warp-cooperative row search (levels 5..10 on inputs > 16 KB).  The lazy control flow stays sequential and is
// executed uniformly by all lanes (same scalars, broadcast loads); what is spread over the lanes is the search itself:
// lane j takes the j-th entry of the row in the reference's visiting order (head, head+1, ... mod rowEntries), the tag
// compare becomes one ballot, every accepted candidate is measured by its own lane, and the winner is the first
// candidate of maximal length -- which is what the serial loop's "strictly longer replaces" rule selects.  Table
// writes are made by lane 0 only.
// The hash cache of a full warp: entry k lives in lane k's register `hc` (no indexed array, hence no local memory), a shuffle reads it;
// narrower groups keep the array.
template <class C>
ZB_HD void row_fill_cache_w(const C& w, RowState& ms, u32 idx, const u8* iLimit) {
    if (C::W < 32) { row_fill_cache(ms, idx, iLimit); return; }
    u32 const maxElems = (ms.base + idx) > iLimit ? 0 : (u32)(iLimit - (ms.base + idx) + 1);
    u32 const lim = idx + (8 < maxElems ? 8 : maxElems);
    u32 const q = idx + (((u32)w.lane - idx) & 7);              // the position of [idx, idx + 8) whose entry this lane holds
    if ((u32)w.lane < 8 && q < lim) { u32 const h = row_hash(ms.base + q, ms.rowHashLog + 8, ms.mls); row_prefetch(ms, h); ms.hc = h; }
}
template <class C>
ZB_HD u32 row_next_cached_w(const C& w, RowState& ms, u32 idx) {
    if (C::W < 32) return row_next_cached(ms, idx);
    u32 const newHash = row_hash(ms.base + idx + 8, ms.rowHashLog + 8, ms.mls);
    row_prefetch(ms, newHash);
    u32 const hash = w.shfl(ms.hc, (int)(idx & 7));
    if ((u32)w.lane == (idx & 7)) ms.hc = newHash;
    return hash;
}
// Positions [from, to) inserted by a whole warp at once, with the result of inserting them one after the other: lanes that hit the
// same row find each other with a match-any vote, the r-th of them takes the r-th step of the row's head (head-1, ..., 1, rowMask,
// ...), the last one leaves the head behind, and where a long run of equal hashes wraps around a row only the latest writer of an
// entry stores.  One memory round trip per 32 positions instead of one per position.
template <class C>
ZB_HD void row_insert_batch(const C& w, RowState& ms, u32 from, u32 to) {
    u32 const rowMask = (1u << ms.rowLog) - 1;
    for (u32 b = from; b < to; b += (u32)C::W) {
        u32 const i = b + (u32)w.lane;
        bool const active = i < to;
        u32 const hash = active ? row_hash(ms.base + i, ms.rowHashLog + 8, ms.mls) : 0;
        u32 const relRow = (hash >> 8) << ms.rowLog;
        u8* const tagRow = ms.tagTable + relRow;
        u32 const grp = w.match_any(active ? relRow : (0x80000000u | (u32)w.lane));
        u32 const rank = popc32(grp & ((1u << w.lane) - 1)), cnt = popc32(grp);
        u32 h = active ? ((u32)*tagRow & rowMask) : 1u;
        h = h ? h : 1u;                                        // an empty row's first entry is rowMask, like a head of 1
        w.sync();                                              // every lane has read its row's head
        if (active) {
            u32 const pos = (h + 4 * rowMask - 2 - rank) % rowMask + 1;
            if (rank + rowMask >= cnt) { tagRow[pos] = (u8)hash; ms.hashTable[relRow + pos] = i; }
            if (rank + 1 == cnt) *tagRow = (u8)pos;
        }
        w.sync();
    }
}
template <class C>
ZB_HD void row_update_warp(const C& w, RowState& ms, const u8* ip) {
    u32 idx = ms.nextToUpdate;
    u32 const target = (u32)(ip - ms.base);
    u32 const rowMask = (1u << ms.rowLog) - 1;
    auto insert_range = [&](u32 from, u32 to) {
        for (u32 i = from; i < to; ++i) {
            u32 const hash = row_next_cached_w(w, ms, i);     // uniform
            if (w.lane == 0) {
                u32 const relRow = (hash >> 8) << ms.rowLog;
                u8* const tagRow = ms.tagTable + relRow;
                u32 const pos = row_next_index(tagRow, rowMask);
                tagRow[pos] = (u8)hash;
                ms.hashTable[relRow + pos] = i;
            }
        }
    };
    if (C::W >= 32 && target - idx > 2) {
        // the hash cache holds nothing but row_hash() of the next eight positions, so the batch works from the hashes themselves and
        // the cache is brought to where the serial walk would have left it: positions target .. target + 7
        if (target - idx > 384) { row_insert_batch(w, ms, idx, idx + 96); idx = target - 32; }
        row_insert_batch(w, ms, idx, target);
        {   u32 const q = target + (((u32)w.lane - target) & 7);
            if ((u32)w.lane < 8) { u32 const h = row_hash(ms.base + q, ms.rowHashLog + 8, ms.mls); row_prefetch(ms, h); ms.hc = h; } }
        ms.nextToUpdate = target;
        return;
    }
    if (target - idx > 384) {
        insert_range(idx, idx + 96);
        idx = target - 32;
        row_fill_cache_w(w, ms, idx, ip + 1);
    }
    insert_range(idx, target);
    ms.nextToUpdate = target;
}
template <class C>
ZB_HD size_t row_find_best_warp(const C& w, RowState& ms, const u8* ip, const u8* iLimit, size_t* offBasePtr) {
    u32 const curr = (u32)(ip - ms.base);
    u32 const lowLimit = 2;
    u32 const rowEntries = 1u << ms.rowLog, rowMask = rowEntries - 1;
    u32 const maxAttempts = 1u << (ms.searchLog < ms.rowLog ? ms.searchLog : ms.rowLog);
    u32 hash;
    if (!ms.lazySkipping) { row_update_warp(w, ms, ip); hash = row_next_cached_w(w, ms, curr); }
    else { hash = row_hash(ip, ms.rowHashLog + 8, ms.mls); ms.nextToUpdate = curr; }
    w.sync();                                              // lane 0's insertions are visible to everybody
    u32 const relRow = (hash >> 8) << ms.rowLog;
    u32 const tag = hash & 0xFF;
    u32* const row = ms.hashTable + relRow;
    u8* const tagRow = ms.tagTable + relRow;
    // a full warp fetches the tag row and the index row in ONE round trip -- lane e holds entries e (and e + 32) -- and the visiting
    // order (head, head + 1, ... mod rowEntries) is a shuffle; narrower groups walk the rows as the serial code does
    u32 tb0 = 0, tb1 = 0, ix0 = 0, ix1 = 0;
    if (C::W >= 32) {
        if ((u32)w.lane < rowEntries) { tb0 = tagRow[w.lane]; ix0 = row[w.lane]; }
        if (rowEntries > 32) { tb1 = tagRow[32 + w.lane]; ix1 = row[32 + w.lane]; }
    }
    u32 const head = (C::W >= 32 ? w.shfl(tb0, 0) : (u32)*tagRow) & rowMask;
    u32 const ip4 = load32(ip);
    u32 bestLen = 0, bestIdx = 0; bool stopped = false; u32 used = 0;
    for (u32 base = 0; base < rowEntries && !stopped && used < maxAttempts; base += (u32)C::W) {
        u32 const j = base + (u32)w.lane;
        u32 const matchPos = (head + j) & rowMask;
        bool hit; u32 idx;
        if (C::W >= 32) {
            int const from = (int)(matchPos & 31);
            u32 const t0 = w.shfl(tb0, from), x0 = w.shfl(ix0, from);
            u32 t = t0, x = x0;
            if (rowEntries > 32) { u32 const t1 = w.shfl(tb1, from), x1 = w.shfl(ix1, from); if (matchPos >> 5) { t = t1; x = x1; } }
            hit = j < rowEntries && matchPos != 0 && t == tag;
            idx = hit ? x : 0;
        } else {
            hit = j < rowEntries && matchPos != 0 && tagRow[matchPos] == (u8)tag;
            idx = hit ? row[matchPos] : 0;
        }
        u32 const hitMask = w.ballot(hit), staleMask = w.ballot(hit && idx < lowLimit);
        u32 valid = hitMask;
        if (staleMask) { valid &= (1u << ctz32(staleMask)) - 1; stopped = true; }
        u32 const rank = used + popc32(valid & ((1u << w.lane) - 1));
        bool const mine = ((valid >> w.lane) & 1) && rank < maxAttempts;
        u32 len = 0;
        if (mine) { const u8* const match = ms.base + idx; if (load32(match) == ip4) len = (u32)count_match(ip, match, iLimit); }
        u32 const lmax = w.max(len);
        if (lmax > bestLen && lmax >= 4) {                 // strictly longer than everything before: first lane holding it wins
            u32 const who = ctz32(w.ballot(mine && len == lmax));
            bestLen = lmax; bestIdx = w.shfl(idx, (int)who);
        }
        used += popc32(valid);
    }
    w.sync();
    if (w.lane == 0) {                                     // "insert current byte into hashtable too" (row_next_index from the head read above)
        u32 pos = (head - 1) & rowMask; pos += pos == 0 ? rowMask : 0;
        tagRow[0] = (u8)pos; tagRow[pos] = (u8)tag;
        row[pos] = ms.nextToUpdate;
    }
    ms.nextToUpdate++;
    w.sync();
    if (bestLen >= 4) { *offBasePtr = (size_t)(curr - bestIdx) + 3; return bestLen; }
    return 3;
}
template <class C>
ZB_HDN u32 parse_lazy_warp(const C& w, const EncWork& W, const u8* src, size_t srcSize, u32 hashLog, u32 searchLog, u32 minMatch, u32 depth, u32* lastLL) {
    bool const useRow = true; u32 const finder = 1, chainLog = 0;
    const u8* const istart = src;
    const u8* ip = istart;
    const u8* anchor = istart;
    const u8* const iend = istart + srcSize;
    const u8* const ilimit = useRow ? iend - 8 - 8 : iend - 8;
    const u8* const prefixLowest = src;
    u32 offset_1 = 1, offset_2 = 4, nbSeq = 0;
    // repcode matches are measured by the whole group (ZSTD_count of two uniform pointers)
    auto wc = [&](const u8* a, const u8* b) { return (size_t)wcount(w, src, (u32)srcSize, (u32)(a - src), (u32)(b - src)); };
    RowState ms;
    ms.finder = finder; ms.chainTable = W.hashSmall; ms.hashLog = hashLog; ms.chainLog = chainLog;
    ms.hashTable = W.hashLong; ms.tagTable = reinterpret_cast<u8*>(W.hashSmall); ms.base = src - 2;
    ms.mls = minMatch < 4 ? 4 : minMatch > 6 ? 6 : minMatch;
    ms.rowLog = searchLog < 4 ? 4 : searchLog > 6 ? 6 : searchLog;
    ms.searchLog = searchLog; ms.rowHashLog = hashLog - ms.rowLog;
    ms.nextToUpdate = 2; ms.lazySkipping = false; ms.hc = 0;
    ip += 1;
    {   u32 const maxRep = (u32)(ip - prefixLowest);
        if (offset_2 > maxRep) offset_2 = 0;
        if (offset_1 > maxRep) offset_1 = 0; }
    if (useRow) row_fill_cache_w(w, ms, ms.nextToUpdate, ilimit);
    while (ip < ilimit) {
        size_t matchLength = 0;
        size_t offBase = 1;
        const u8* start = ip + 1;
        bool store = false;
        if ((offset_1 > 0) && (load32(ip + 1 - offset_1) == load32(ip + 1))) {
            matchLength = wc(ip + 1 + 4, ip + 1 + 4 - offset_1) + 4;
            if (depth == 0) store = true;
        }
        if (!store) {
            // The searches at ip, ip + 1 (lazy) and ip + 2 (lazy2) of zstd_lazy.c:1581-1660 as ONE call site in a small state machine
            // (stage = which of the three is due), so that the finder is inlined once: three copies of it do not fit the
            // instruction cache next to each other.
            u32 stage = 0; bool found = true;
            for (;;) {
                if (stage) {
                    ip++;
                    if ((offBase) && ((offset_1 > 0) && (load32(ip) == load32(ip - offset_1)))) {
                        size_t const mlRep = wc(ip + 4, ip + 4 - offset_1) + 4;
                        int const mul = stage == 1 ? 3 : 4;
                        int const gain2 = (int)(mlRep * mul);
                        int const gain1 = (int)(matchLength * mul - highbit32((u32)offBase) + 1);
                        if ((mlRep >= 4) && (gain2 > gain1)) { matchLength = mlRep; offBase = 1; start = ip; }
                    }
                }
                size_t ofb = 999999999;
                size_t const ml2 = row_find_best_warp(w, ms, ip, iend, &ofb);
                if (stage == 0) {
                    if (ml2 > matchLength) { matchLength = ml2; start = ip; offBase = ofb; }
                    if (matchLength < 4) { found = false; break; }
                    if (depth == 0 || !(ip < ilimit)) break;
                    stage = 1; continue;
                }
                int const gain2 = (int)(ml2 * 4 - highbit32((u32)ofb));
                int const gain1 = (int)(matchLength * 4 - highbit32((u32)offBase) + (stage == 1 ? 4 : 7));
                if ((ml2 >= 4) && (gain2 > gain1)) {
                    matchLength = ml2; offBase = ofb; start = ip;
                    if (!(ip < ilimit)) break;
                    stage = 1; continue;
                }
                if (stage == 1 && depth == 2 && ip < ilimit) { stage = 2; continue; }
                break;
            }
            if (!found) {
                size_t const step = ((size_t)(ip - anchor) >> 8) + 1;      // kSearchStrength
                ip += step;
                ms.lazySkipping = step > 8;                                // kLazySkippingStep
                continue;
            }
            if (offBase > 3) {   // catch up
                size_t const off = offBase - 3;
                while (((start > anchor) && (start - off > prefixLowest)) && (start[-1] == (start - off)[-1])) { start--; matchLength++; }
                offset_2 = offset_1; offset_1 = (u32)off;
            }
        }
        if (w.lane == 0) { W.put(nbSeq, (u32)(start - anchor), (u32)offBase, (u32)matchLength); }
        nbSeq++;
        anchor = ip = start + matchLength;
        if (ms.lazySkipping) { if (useRow) row_fill_cache_w(w, ms, ms.nextToUpdate, ilimit); ms.lazySkipping = false; }
        while (((ip <= ilimit) && (offset_2 > 0)) && (load32(ip) == load32(ip - offset_2))) {
            matchLength = wc(ip + 4, ip + 4 - offset_2) + 4;
            u32 const tmp = offset_2; offset_2 = offset_1; offset_1 = tmp;
            if (w.lane == 0) { W.put(nbSeq, 0, 1, (u32)matchLength); }
            nbSeq++;
            ip += matchLength; anchor = ip;
        }
    }
    w.sync();
    *lastLL = (u32)(iend - anchor);
    return nbSeq;
}

// ------------------------------------------------------------------ sequence export
// The parse of one block in the layout of the reference's public ZSTD_Sequence (N/zstd.h:1315-1350), as
// ZSTD_generateSequences / ZSTD_copyBlockSequences (N/compress/zstd_compress.c:3429-3512) write it for the first block of
// a frame (repcode history {1,4,8}): one record per sequence with the raw offset and the `rep` field resolved, then one
// {offset 0, litLength = trailing literals, matchLength 0} record -- the block delimiter.  This is also what an external
// sequence producer (ZSTD_sequenceProducer_F, N/zstd.h:2820-2900) hands back to libzstd.
// Rows of W sequences: loads and stores are one 16-byte record per lane; the repcode history is a serial scan that
// every lane follows with shuffles (three registers), lane k keeping the offset of its own sequence.
// A block the reference would not parse (srcSize < 7, PARSE_SKIPPED) is exported as literals only.  Returns the number
// of records (uniform), at most MAX_SEQ + 1.
struct alignas(16) ZSeq { u32 offset, litLength, matchLength, rep; };
template <class C>
ZB_HDN u32 export_sequences(const C& w, const Seq* in, u32 nbSeq, u32 lastLL, size_t srcSize, ZSeq* out) {
    if (nbSeq == PARSE_SKIPPED) { nbSeq = 0; lastLL = (u32)srcSize; }
    u32 rep0 = 1, rep1 = 4, rep2 = 8;
    for (u32 base = 0; base < nbSeq; base += C::W) {
        u32 const i = base + (u32)w.lane;
        Seq q; q.ll = 0; q.of = 0; q.ml = 0; q.pad = 0;
        if (i < nbSeq) q = in[i];
        u32 const rows = (nbSeq - base < (u32)C::W) ? nbSeq - base : (u32)C::W;
        u32 raw = 0, repField = 0;
        for (u32 k = 0; k < rows; k++) {
            u32 const of = w.shfl(q.of, (int)k), ll0 = w.shfl(q.ll, (int)k) == 0 ? 1u : 0u;
            u32 r, f = 0;
            if (of > 3) { r = of - 3; rep2 = rep1; rep1 = rep0; rep0 = r; }
            else {                                             // repcode 1..3 (ZSTD_updateRep, zstd_compress_internal.h:817-835)
                f = of;
                u32 const rc = of - 1 + ll0;
                r = rc == 0 ? rep0 : rc == 1 ? rep1 : rc == 2 ? rep2 : rep0 - 1;
                if (rc > 0) { if (rc >= 2) rep2 = rep1; rep1 = rep0; rep0 = r; }
            }
            if ((u32)w.lane == k) { raw = r; repField = f; }
        }
        if (i < nbSeq) { ZSeq z; z.offset = raw; z.litLength = q.ll; z.matchLength = q.ml; z.rep = repField; out[i] = z; }
    }
    if (w.lane == 0) { ZSeq z; z.offset = 0; z.litLength = lastLL; z.matchLength = 0; z.rep = 0; out[nbSeq] = z; }
    w.sync();
    return nbSeq + 1;
}

// ------------------------------------------------------------------ frame
// A chunk becomes a frame in two stages that may run in different kernels (and with different group widths):
//   parse_stage   match finding -> sequences (W.seq*), their count and the trailing literal run
//   encode_stage  frame/block headers, literal gathering, Huffman + FSE entropy stage
// Together they emit what ZSTD_compress2 would with dstCapacity = ZSTD_compressBound(srcSize).
constexpr u32 FRAME_CHECKSUM = 1, FRAME_NO_CONTENT_SIZE = 2, FRAME_MAGICLESS = 4;      // frameFlags: ZSTD_c_checksumFlag = 1, ZSTD_c_contentSizeFlag = 0, ZSTD_c_format = ZSTD_f_zstd1_magicless

// ONLY = 0: every parser is compiled in.  ONLY = S_dfast / S_fast: the caller guarantees that this level selects that
// strategy for every input size, so the kernel holds a single cooperative parser (64 registers without spills; the
// all-in-one instantiation needs ~1 KB of stack).  ONLY = ONLY_LAZY: greedy ... btlazy2 for every input size (levels 5 and up):
// the cooperative row-based parser plus the serial finders, built with its own register budget.
constexpr u32 ONLY_LAZY = 64;
template <class C, u32 ONLY = 0>
ZB_HDN size_t parse_stage(const C& w, const EncWork& W, const u8* src, size_t srcSize, int level, u32* nbSeqOut, u32* lastLLOut, const CParams* ov = nullptr) {
    CParams cp;
    *nbSeqOut = PARSE_SKIPPED; *lastLLOut = 0;
    if (!get_cparams(&cp, level, srcSize, ov)) return ERR(E_parameter_unsupported);
    if (ONLY == ONLY_LAZY ? cp.strategy < S_greedy : (ONLY != 0 && cp.strategy != ONLY)) return ERR(E_GENERIC);
    if (srcSize < 7) return 0;
    {   // fresh tables: zero the used part (16-byte stores; the workspace is 16-byte aligned)
        u32 const nL = (1u << cp.hashLog) / 4;
        u32 const nS = (cp.strategy == S_dfast) ? (1u << cp.chainLog) / 4                               // short-hash table
                     : (cp.strategy >= S_greedy) ? ((cp.strategy != S_btlazy2 && cp.windowLog > 14) ? (1u << cp.hashLog) / 16   // tag bytes of the row finder
                                                                        : (1u << cp.chainLog) / 4) : 0;  // chain table / binary tree
        struct alignas(16) Q { u32 a, b, c, d; };
        Q* const qL = reinterpret_cast<Q*>(W.hashLong); Q* const qS = reinterpret_cast<Q*>(W.hashSmall);
        Q const z = { 0, 0, 0, 0 };
        for (u32 i = (u32)w.lane; i < nL; i += C::W) qL[i] = z;
        for (u32 i = (u32)w.lane; i < nS; i += C::W) qS[i] = z;
        w.sync(); }
    u32 nbSeq = 0, lastLL = 0;
    if (C::W > 1 && (ONLY == S_dfast || (ONLY == 0 && cp.strategy == S_dfast))) {
        if (ONLY == S_dfast && cp.minMatch == 5) nbSeq = parse_dfast_warp<C, 5>(w, W, src, srcSize, cp.hashLog, cp.chainLog, 5, &lastLL);
        else nbSeq = parse_dfast_warp(w, W, src, srcSize, cp.hashLog, cp.chainLog, cp.minMatch, &lastLL);
    } else if (C::W > 1 && (ONLY == S_fast || (ONLY == 0 && cp.strategy == S_fast))) {
        nbSeq = parse_fast_warp(w, W, src, srcSize, cp.hashLog, cp.minMatch, cp.targetLength, &lastLL);
    } else if ((ONLY == 0 || ONLY == ONLY_LAZY) && C::W > 1 && cp.strategy >= S_greedy && cp.strategy <= S_lazy2 && cp.windowLog > 14) {
        nbSeq = parse_lazy_warp(w, W, src, srcSize, cp.hashLog, cp.searchLog, cp.minMatch, cp.strategy - S_greedy, &lastLL);
    } else if (ONLY == 0 || ONLY == ONLY_LAZY) {
        if (w.lane == 0) {
            if (ONLY == ONLY_LAZY || cp.strategy >= S_greedy) nbSeq = parse_lazy(W, src, srcSize, cp.hashLog, cp.chainLog, cp.searchLog, cp.minMatch, cp.strategy == S_btlazy2 ? 2 : cp.strategy - S_greedy,
                                                          cp.strategy == S_btlazy2 ? 2u : cp.windowLog > 14 ? 1u : 0u, &lastLL);
            else if (cp.strategy == S_dfast) nbSeq = parse_dfast(W, src, srcSize, cp.hashLog, cp.chainLog, cp.minMatch, &lastLL);
            else nbSeq = parse_fast(W, src, srcSize, cp.hashLog, cp.minMatch, cp.targetLength, &lastLL);
        }
        w.sync();
        nbSeq = w.bcast(nbSeq); lastLL = w.bcast(lastLL);
    }
    *nbSeqOut = nbSeq; *lastLLOut = lastLL;
    return 0;
}

// `dst` must have room for compress_bound(srcSize) + 32 bytes.  Uniform return value.
template <class C>
ZB_HDN size_t encode_stage(const C& w, EncShared& S, const EncWork& W, u8* dst, size_t dstCapacity, const u8* src, size_t srcSize, int level, u32 nbSeq, u32 lastLL,
                           u32 frameFlags = 0, const CParams* ov = nullptr) {
    CParams cp;
    if (!get_cparams(&cp, level, srcSize, ov)) return ERR(E_parameter_unsupported);
    if (dstCapacity < 18) return ERR(E_dstSize_tooSmall);
    size_t pos = 0;
    // ZSTD_writeFrameHeader :4695-4743 (no dictionary): the pledged size is known in a one-shot call, so the window
    // covers the input and the frame is "single segment" whenever the content size is written
    bool const checksum = (frameFlags & FRAME_CHECKSUM) != 0, contentSize = !(frameFlags & FRAME_NO_CONTENT_SIZE);
    u32 const fcsCode = contentSize ? (srcSize >= 256) + (srcSize >= 65536 + 256) : 0;
    u32 const mlen = (frameFlags & FRAME_MAGICLESS) ? 0u : 4u;        // the magic number is written for ZSTD_f_zstd1 only (:4716-4719)
    if (w.lane == 0) {
        if (mlen) { dst[0] = 0x28; dst[1] = 0xB5; dst[2] = 0x2F; dst[3] = 0xFD; }
        u8* const h = dst + mlen;
        h[0] = (u8)((checksum ? 4 : 0) + (contentSize ? (1 << 5) : 0) + (fcsCode << 6));
        if (!contentSize) h[1] = (u8)((cp.windowLog - 10) << 3);
        else if (fcsCode == 0) h[1] = (u8)srcSize;
        else if (fcsCode == 1) { u32 const v = (u32)srcSize - 256; h[1] = (u8)v; h[2] = (u8)(v >> 8); }
        else { u32 const v = (u32)srcSize; h[1] = (u8)v; h[2] = (u8)(v >> 8); h[3] = (u8)(v >> 16); h[4] = (u8)(v >> 24); }
    }
    pos = mlen + 1 + (!contentSize ? 1 : fcsCode == 0 ? 1 : fcsCode == 1 ? 2 : 4);
    // ZSTD_writeEpilogue :5344-5381: the low 32 bits of XXH64(content) follow the last block when asked for
    u32 const sumBytes = checksum ? 4 : 0;
    u32 sum = 0;
    if (checksum && w.lane == 0) sum = (u32)xxh64(src, srcSize);
    if (srcSize == 0) {   // :5364-5372
        if (dstCapacity - pos < 3 + sumBytes) return ERR(E_dstSize_tooSmall);
        if (w.lane == 0) { dst[pos] = 1; dst[pos + 1] = 0; dst[pos + 2] = 0;
                           if (checksum) { dst[pos + 3] = (u8)sum; dst[pos + 4] = (u8)(sum >> 8); dst[pos + 5] = (u8)(sum >> 16); dst[pos + 6] = (u8)(sum >> 24); } }
        w.sync();
        return pos + 3 + sumBytes;
    }
    u8* const op = dst + pos; size_t const cap = dstCapacity - pos;
    ZB_PT_DECL
    if (cap < 3 + 2 + 1) return ERR(E_dstSize_tooSmall);
    size_t cSize = 0;
    if (nbSeq != PARSE_SKIPPED) {
        // gather literals (ZSTD_storeSeq copies them during the parse; the result is the same buffer)
        size_t litSize = 0;
        {   // 32 sequences per step: source / literal positions by prefix sums, short runs copied by the lane that
            // owns the sequence, long runs by the whole group
            size_t sp = 0;
            for (u32 base = 0; base < nbSeq; base += C::W) {
                u32 const i = base + (u32)w.lane;
                Seq q; q.ll = 0; q.of = 0; q.ml = 0; q.pad = 0;
                if (i < nbSeq) q = W.get(i);
                u32 const ll = q.ll, ml = q.ml;
                u32 const lpre = w.exscan(ll), spre = w.exscan(ll + ml);
                if (ll && ll <= 32) copy_fwd(W.lit + litSize + lpre, src + sp + spre, ll);
                u32 big = w.ballot(ll > 32);
                while (big) {
                    int const b = (int)ctz32(big); big &= big - 1;
                    u32 const L = w.shfl(ll, b), lp = w.shfl(lpre, b), spp = w.shfl(spre, b);
                    u8* const d = W.lit + litSize + lp; const u8* const f = src + sp + spp;
                    for (u32 k = (u32)w.lane; k < L; k += C::W) d[k] = f[k];
                }
                litSize += w.bcast(lpre + ll, C::W - 1); sp += w.bcast(spre + ll + ml, C::W - 1);
            }
            for (u32 j = (u32)w.lane; j < lastLL; j += C::W) W.lit[litSize + j] = src[sp + j];
            litSize += lastLL;
            w.sync(); }
        ZB_PT(1);      // literal gather
        bool const disableLit = (cp.strategy == S_fast && cp.targetLength > 0);   // ZSTD_literalsCompressionIsDisabled
        cSize = entropy_compress(w, S, W, op + 3, cap - 3, nbSeq, litSize, cp.strategy, disableLit);
        // ZSTD_entropyCompressSeqStore_wExtLitBuffer :3005-3042
        if (cSize == ERR(E_dstSize_tooSmall) && srcSize <= cap - 3) cSize = 0;
        if (isErr(cSize)) return cSize;
        if (cSize) { size_t const maxCSize = srcSize - ((srcSize >> 6) + 2); if (cSize >= maxCSize) cSize = 0; }
    }
    if (cSize == 0) {   // ZSTD_noCompressBlock
        if (srcSize + 3 > cap) return ERR(E_dstSize_tooSmall);
        if (w.lane == 0) { u32 const h = 1 + (u32)(srcSize << 3); op[0] = (u8)h; op[1] = (u8)(h >> 8); op[2] = (u8)(h >> 16); }
        wcopy(w, op + 3, src, srcSize);
        cSize = srcSize;
    } else if (w.lane == 0) { u32 const h = 1 + (2 << 1) + (u32)(cSize << 3); op[0] = (u8)h; op[1] = (u8)(h >> 8); op[2] = (u8)(h >> 16); }
    if (checksum) {
        if (cap - (3 + cSize) < 4) return ERR(E_dstSize_tooSmall);
        if (w.lane == 0) { u8* const q = op + 3 + cSize; q[0] = (u8)sum; q[1] = (u8)(sum >> 8); q[2] = (u8)(sum >> 16); q[3] = (u8)(sum >> 24); }
    }
    w.sync();
    return pos + 3 + cSize + sumBytes;
}

// both stages on one context (host instantiation, single-kernel use)
template <class C>
ZB_HDN size_t compress_frame(const C& w, EncShared& S, const EncWork& W, u8* dst, size_t dstCapacity, const u8* src, size_t srcSize, int level, u32 frameFlags = 0,
                             const CParams* ov = nullptr) {
    u32 nbSeq = 0, lastLL = 0;
    size_t const r = parse_stage(w, W, src, srcSize, level, &nbSeq, &lastLL, ov);
    if (isErr(r)) return r;
    return encode_stage(w, S, W, dst, dstCapacity, src, srcSize, level, nbSeq, lastLL, frameFlags, ov);
}

}  // namespace zb
