// zb_decode_fast.cuh -- staged ("transposed") decoder for batches of single-block frames, second generation.
//
// In a batch of thousands of frames the serial chains of the format (Huffman streams, the three coupled FSE
// states of the sequence stream) are the critical path.  This pipeline gives every chain its own *thread*, runs
// all of them at once next to each other, and then executes the sequences with whole warps:
//
//   A  dec_prepare   warp / frame    frame_walk: one frame of one block; prepare_block (shared with the segment decoder): section
//                                    headers, Huffman and FSE decode tables -> HBM, bit lengths of every backward stream
//   B  HufChain      thread / stream 4 x n chains, each decodes one Huffman stream into the literal buffer   } one persistent
//   C  SeqChain      thread / frame  sequence bitstream -> (litLength, matchLength, offset) packed in 8 B   } kernel (k_dec_chains)
//   D  dec_exec      warp / frame    "byte gather": every output byte finds its sequence and its source byte,
//                                    128 output bytes per round, no ordering between the lanes
//
// Both chain kinds read their bitstream through a `word source`: on the GPU a per-lane ring in shared memory that
// 16-byte asynchronous copies (cp.async) keep several hundred bytes ahead of the reader, on the host (tests) the
// plain byte array.  Their tables sit in shared memory, brought in by one bulk asynchronous copy
// (cp.async.bulk + mbarrier) per table when a lane takes its next frame.
//
// An item is eligible when it is exactly one frame with one (last) block and carries its content size; a checksum is
// verified at the end of stage D by the warp (xxh64_warp).  Everything else (multi-block, skippable, > MAXS sequences,
// 2^12-cell Huffman tables) is left to the fused kernel or the segment decoder; an item of several frames is cut into
// its frames first (item_walk, the decode list of the host-memory calls).  Results -- including the error code of corrupted input --
// are identical to the fused path: the stage statuses are combined in the order the fused decoder would have met the errors.
//
// Reference behaviour reproduced: see zb_decode.cuh (N/decompress/zstd_decompress_block.c:134-340,695-775,
// 1001-1096,1229-1346,1615-1690; N/decompress/huf_decompress.c:574-698).
#pragma once
#include "zb_decode.cuh"

namespace zb {

constexpr u32 FAST_MAXS = 43776;            // > 131072 / MINMATCH: more sequences cannot fit a 128 KB block
constexpr u32 FAST_HUF_LOG = 11;            // largest Huffman table the staged path takes (the reference never writes 2^12)
constexpr u32 FAST_HUF_ENTRIES = 1u << FAST_HUF_LOG;
constexpr u32 FAST_FSE_ENTRIES = 512 + 256 + 512;  // LL | OF | ML
constexpr u32 FAST_FSE_OF = 512, FAST_FSE_ML = 768;
// FSE table t (0 LL, 1 OF, 2 ML) of a frame's or a block's FAST_FSE_ENTRIES cells: cells [fse_at(t), fse_at(t + 1))
ZB_HD u32 fse_at(int t) { constexpr u32 at[4] = { 0, FAST_FSE_OF, FAST_FSE_ML, FAST_FSE_ENTRIES }; return at[t]; }
constexpr u32 NO_END_MARK = 0xFFFFFFFFu;

// Bits of the backward stream p[0, len) below its end mark, the highest set bit of its last byte.  NO_END_MARK: the stream is empty or
// its last byte is zero, which BIT_initDStream (HUF_decompress1X1, ZSTD_decompressSequences) rejects as corruption.
ZB_HD u32 end_mark_bits(const u8* p, u32 len) {
    u32 const last = len ? p[len - 1] : 0u;
    return last ? (len - 1) * 8 + highbit32(last) : NO_END_MARK;
}

// FSE cell of the staged path: extra bits of the code (bits 0..7) | nbBits (8..15) | new-state base (16..24) | code (25..30).
// The byte-aligned bit counts make the sum of the three cells of a sequence carry both totals at once
// (byte 0: offset + matchLength + litLength extra bits <= 63, byte 1: state bits <= 26).
ZB_HD u32 fse2_pack(u32 e, u32 extra) { return extra | (((e >> 16) & 0xFF) << 8) | ((e & 0x1FF) << 16) | ((e >> 24) << 25); }

struct DecDesc {
    u32 mode;            // 0 = not eligible (fused kernel handles the item), 1 = compressed block, 2 = raw block, 3 = rle block
    u32 stA1, stB, stA2, stC, stD;   // positive error codes per stage (0 = fine)
    u32 blockOff, cSize; // block content inside the item
    u32 contentSize;
    u32 litMode, litSize, rawOff, rleByte, hufLog, nStreams;
    u32 sOff[4], sLen[4], oOff[4], oCnt[4];      // relative to the block content / the literal buffer
    u32 sBits[4];                                // bits of Huffman stream k below its end mark (NO_END_MARK: none)
    u32 nbSeq, seqOff, seqLen;                   // sequence bitstream inside the block content
    u32 seqBits;                                 // bits of the sequence stream below its end mark
    union {                                      // the three FSE table logs, by table index or by name
        u32 fseLog[3];
        struct { u32 logLL, logOF, logML; };
    };
    u32 regen;
    u32 hufLitSize;      // litSize when the literals are Huffman coded, else 0 (sort key of the Huffman chains)
    u32 seqUnusable;     // the sequence stream has no end mark: stC is final, nothing is decoded or executed
    u32 outMax;          // most bytes the compressed block may write (block_output_limit), 0xFFFFFFFF: the capacity
};
// k_dec_chains and k_order read these fields (k_order through a stride of sizeof(DecDesc) / 4): keeping the layout keeps their code
static_assert(sizeof(DecDesc) == 184 && offsetof(DecDesc, sBits) == 124 && offsetof(DecDesc, nbSeq) == 140 && offsetof(DecDesc, seqBits) == 152 &&
              offsetof(DecDesc, fseLog) == 156 && offsetof(DecDesc, hufLitSize) == 172 && offsetof(DecDesc, seqUnusable) == 176, "DecDesc layout");

// ---------------------------------------------------------------------------------------- stage A
// The blocks of an item that is exactly one frame of at most maxBlocks blocks: magic number (none when magicless), no dictionary, every
// block inside the item, the checksum (when the frame has one) its last four bytes.  Returns the number of blocks (0: the item is not
// such a frame); refs[k] = offset of block k's header | that header << 32 (refs may be null), *xxh = the stored checksum.
// With `end`, the frame only has to start the item: *end = its size (frames past 4 GiB are not taken).
ZB_HDN u32 frame_walk(const u8* src, size_t size, FrameHeader* fh, u32 maxBlocks, u64* refs, u32* xxh, size_t* end = nullptr, u32 magicless = 0) {
    if (end && size > 0xFFFFFFFFu) size = 0xFFFFFFFFu;
    if (size < (magicless ? 5u : 9u) || size > 0xFFFFFFFFu || (!magicless && load32(src) != MAGIC)) return 0;
    if (read_frame_header(fh, src, size, magicless) != 0 || fh->skippable || fh->dictID) return 0;
    size_t pos = fh->headerSize; u32 n = 0;
    for (;;) {
        if (size - pos < 3 || n == maxBlocks) return 0;
        u32 const bh = load24(src + pos), type = (bh >> 1) & 3;
        size_t const cSize = type == 1 ? 1 : bh >> 3;
        if (type == 3 || cSize > size - pos - 3) return 0;
        if (refs) refs[n] = (u64)pos | ((u64)bh << 32);
        n++; pos += 3 + cSize;
        if (bh & 1) break;
    }
    size_t const tail = fh->checksum ? 4u : 0u;
    if (end ? size - pos < tail : size - pos != tail) return 0;
    *xxh = fh->checksum ? load32(src + pos) : 0;
    if (end) *end = pos + tail;
    return n;
}

// One frame of an item as item_walk lists it.
struct ItemFrame { u64 srcOff, srcSize, contentSize; u32 nBlocks, checksum, hasContentSize, skippable; };

// The frames of an item, for decoding them one by one: frame_walk for each zstd frame, read_frame_header for each skippable one (it
// regenerates nothing).  Lists the frames walked from the item's start into out[0 .. outMax) (out may be null) and returns their number;
// the walk stops where no whole frame follows.  *split: the item may be decoded frame by frame -- the walk covers it exactly, it has at
// least two frames (skippable ones count), every zstd frame but the last declares its content size, and the declared sizes add up to
// at most `capacity` (the last zstd frame, if it declares none, gets the rest).  Any other item is decoded whole.
// A magicless item has no skippable frames: bytes that read like a skippable magic number start a frame there, as in the reference
// (N/decompress/zstd_decompress.c:744,1120).
// *regen (may be null): what the frames of a splittable item regenerate -- their declared sizes, or all of `capacity` when the last zstd
// frame declares none; *mostBlocks (may be null): the most blocks of one of the frames walked.
ZB_HDN u32 item_walk(const u8* src, size_t size, u64 capacity, ItemFrame* out, u32 outMax, bool* split, u32 magicless = 0,
                     u64* regen = nullptr, u32* mostBlocks = nullptr) {
    u32 most = 0;
    u32 n = 0; size_t pos = 0; u64 declared = 0;
    bool sized = true, ok = true;      // sized: every zstd frame so far declares its content size
    while (pos < size) {
        ItemFrame f{}; FrameHeader fh;
        f.srcOff = pos;
        size_t const rest = size - pos;
        if (!magicless && rest >= 8 && (load32(src + pos) & 0xFFFFFFF0u) == 0x184D2A50u) {
            if (read_frame_header(&fh, src + pos, rest) != 0 || (u64)fh.skipLen + 8 > rest) break;
            f.srcSize = 8 + (u64)fh.skipLen; f.skippable = 1;
        } else {
            size_t end = 0; u32 xxh;
            u32 const nb = frame_walk(src + pos, rest, &fh, 0xFFFFFFFFu, nullptr, &xxh, &end, magicless);
            if (!nb) break;
            if (!sized) ok = false;                  // a zstd frame after one without a content size
            f.srcSize = end; f.nBlocks = nb; f.checksum = fh.checksum; f.hasContentSize = fh.hasContentSize; f.contentSize = fh.contentSize;
            if (fh.hasContentSize) declared += fh.contentSize <= capacity ? fh.contentSize : capacity + 1;      // (no wrap)
            else sized = false;
            most = nb > most ? nb : most;
        }
        if (out && n < outMax) out[n] = f;
        n++; pos += (size_t)f.srcSize;
    }
    *split = ok && pos == size && n >= 2 && declared <= capacity;
    if (regen) *regen = sized ? declared : capacity;
    if (mostBlocks) *mostBlocks = most;
    return n;
}

// One block of an item (both decoders): `bh` = its header, at item + off.  Describes it in L -- raw / rle, or for a compressed block the
// literal geometry, the Huffman and sequence stream bits, the stage statuses, seqUnusable and outMax -- and copies out the tables the
// block itself describes: the Huffman table when the literals carry one, every FSE table that is not a repeat.  Whether a repeat is
// legal is the caller's S.litEntropy / S.fseEntropy.  Returns false, the block not described, when its Huffman table is larger than
// 2^hufLogMax (the caller's table stride) or it has more than FAST_MAXS sequences.
template <class C>
ZB_HD bool prepare_block(const C& w, DecShared& S, const u8* item, u32 off, u32 bh, u32 blockSizeMax, size_t dstCapacity, u32 hufLogMax,
                         DecDesc& L, u16* hufOut, u32* fseOut) {
    u32 const type = (bh >> 1) & 3, cSize = type == 1 ? 1 : bh >> 3;
    const u8* const blk = item + off + 3;
    L.blockOff = off + 3; L.cSize = cSize;
    if (type == 0) { L.mode = 2; L.regen = cSize; return true; }
    if (type == 1) { L.mode = 3; L.regen = bh >> 3; L.rleByte = blk[0]; return true; }
    // compressed block: from here on errors are recorded as the stage statuses
    L.mode = 1;
    if (cSize > blockSizeMax) { L.stA1 = E_srcSize_wrong; return true; }
    LitInfo li{};
    size_t const lr = parse_literals(w, S, blk, cSize, blockSizeMax, dstCapacity, &li);
    if (isErr(lr)) { L.stA1 = (u32)(0 - lr); return true; }
    bool const tree = (blk[0] & 3) == 2;
    if (tree && S.hufLog > hufLogMax) return false;
    if (dstCapacity > block_output_limit(dstCapacity, blockSizeMax, li.litSize, li.mode == 0 && lr + LIT_MARGIN <= cSize))
        L.outMax = blockSizeMax + (u32)LIT_MARGIN;
    L.litMode = li.mode; L.litSize = li.litSize; L.rawOff = li.rawOff; L.rleByte = li.rleByte; L.nStreams = li.nStreams;
    for (int k = 0; k < 4; k++) { L.sOff[k] = li.sOff[k]; L.sLen[k] = li.sLen[k]; L.oOff[k] = li.oOff[k]; L.oCnt[k] = li.oCnt[k]; }
    if (tree) {
        L.hufLog = S.hufLog;
        for (u32 i = (u32)w.lane; i < (1u << S.hufLog); i += C::W) hufOut[i] = S.huf[i];
    }
    if (li.mode == 2) {
        L.hufLitSize = li.litSize;
        for (u32 k = 0; k < li.nStreams; k++) {
            L.sBits[k] = end_mark_bits(blk + li.sOff[k], li.sLen[k]);
            if (L.sBits[k] == NO_END_MARK) L.stB = E_corruption_detected;
        }
    }
    int nbSeq = 0;
    size_t const hr = parse_seq_section(w, S, blk + lr, cSize - lr, dstCapacity, &nbSeq);
    if (isErr(hr)) { L.stA2 = (u32)(0 - hr); return true; }
    if ((u32)nbSeq > FAST_MAXS) return false;
    L.nbSeq = (u32)nbSeq; L.seqOff = (u32)(lr + hr); L.seqLen = (u32)(cSize - lr - hr);
    if (nbSeq == 0) return true;
    for (int t = 0; t < 3; t++) {
        if (S.fseMode[t] == 3) continue;
        L.fseLog[t] = S.fseLog[t];
        u32* const out = fseOut + fse_at(t);
        for (u32 i = (u32)w.lane; i < (1u << S.fseLog[t]); i += C::W) {
            u32 const e = S.fse[t][i], sym = e >> 24;
            out[i] = fse2_pack(e, t == 0 ? ZB_T.LL_bits[sym] : t == 1 ? sym : ZB_T.ML_bits[sym]);
        }
    }
    u32 const bits = end_mark_bits(blk + L.seqOff, L.seqLen);
    if (bits == NO_END_MARK) { L.stC = E_corruption_detected; L.seqUnusable = 1; }
    else L.seqBits = bits;
    return true;
}

// The staged decoder takes an item that is one frame of one block, with its content size (at most one block); dec_exec verifies the
// checksum when the frame has one.  All lanes of a warp; S is the warp's shared scratch; tables are copied out to hufOut / fseOut.
// magicless: the item is in the ZSTD_f_zstd1_magicless format.
template <class C>
ZB_HDN void dec_prepare(const C& w, DecShared& S, const u8* src, size_t srcSize, size_t dstCapacity, DecDesc* d, u16* hufOut, u32* fseOut,
                        u32 magicless = 0) {
    DecDesc L{};         // built in registers/local, stored by lane 0 at the end; mode 0: the fused kernel decodes the item
    L.outMax = 0xFFFFFFFFu;
    FrameHeader fh; u64 ref; u32 xxh;
    if (frame_walk(src, srcSize, &fh, 1, &ref, &xxh, nullptr, magicless) && fh.hasContentSize && fh.contentSize <= BLOCKSIZE_MAX) {
        L.contentSize = (u32)fh.contentSize;
        if (w.lane == 0) { S.litEntropy = 0; S.fseEntropy = 0; }      // no earlier block: a repeated table is an error
        w.sync();
        // refused: a 2^12-cell Huffman table (legal, never written by the reference) or a pathological sequence count
        if (!prepare_block(w, S, src, (u32)ref, (u32)(ref >> 32), fh.blockSizeMax, dstCapacity, FAST_HUF_LOG, L, hufOut, fseOut)) L.mode = 0;
    }
    w.sync();
    if (w.lane == 0) *d = L;
    w.sync();
}

// ---------------------------------------------------------------------------------------- word sources
// A backward bitstream is addressed in 32-bit words counted from the 16-byte aligned address at or below its first
// byte: word k holds stream bits [32 k, 32 k + 32) of that numbering, the stream's own bits start at bit `floorBit`
// (= 8 x the distance of the first byte from the aligned address).  Words below the first byte read as zero, the
// word holding it is masked -- mirroring the reference's zero-filled container once a backward stream is exhausted
// (N/common/bitstream.h:344-351).
ZB_HD u32 shr_clamp(u32 v, u32 s) {      // v >> s for s in 0..32
#if defined(__CUDA_ARCH__)
    return __funnelshift_rc(v, 0u, s);
#else
    return s >= 32 ? 0u : v >> s;
#endif
}
struct StreamGeom {
    const u32* W;        // aligned base
    int kFirst;          // word holding the first stream byte
    u32 firstMask;       // valid bits of that word
    u32 floorBit;        // bit index of the stream's first bit
    ZB_HD void set(const u8* ip) {
        uintptr_t const a = reinterpret_cast<uintptr_t>(ip);
        W = reinterpret_cast<const u32*>(a & ~(uintptr_t)15);
        u32 const sb = (u32)(a & 15);
        kFirst = (int)(sb >> 2); firstMask = 0xFFFFFFFFu << (8 * (sb & 3)); floorBit = 8 * sb;
    }
    ZB_HD u32 fix(int k, u32 raw) const { return k > kFirst ? raw : (k == kFirst ? raw & firstMask : 0u); }
};
// host / reference word source: straight from memory
struct MemWords {
    StreamGeom g;
    ZB_HD u32 word(int k) const { return k < g.kFirst ? 0u : g.fix(k, g.W[k]); }
    ZB_HD void fetch4(int k, u32& a, u32& b, u32& c, u32& d) const { a = word(k); b = word(k - 1); c = word(k - 2); d = word(k - 3); }
    ZB_HD void advance(int) {}
    ZB_HD u32 raw(int k) const { return word(k); }
    ZB_HD void fetch4_fast(int k, u32& a, u32& b, u32& c, u32& d) const { fetch4(k, a, b, c, d); }
    ZB_HD void advance_fast(int) {}
};

// ---------------------------------------------------------------------------------------- stage C
// One thread per frame: ZSTD_decodeSequence :1229-1346 for every sequence, offsets resolved against the repcode
// history {1,4,8}; sequences are stored as litLength | matchLength << 18 | offset << 36 (each < 2^18 for a block of
// at most 128 KB; larger values can only come from corrupt input and are clamped to 2^18-1 / 2^28-1, which the
// executor rejects exactly like the originals).
// One step = one sequence, branch free: the next 96 bits of the stream are assembled from four words, the three
// cells give every bit count, and the three fields of the sequence (offset bits | length bits | state bits) are cut
// out of that window.  A sequence reads at most 31 + 32 + 26 = 89 bits.
// The step is cut in two so that, on the GPU, two warps can share it: the WALK (states, bit position: the serial chain proper)
// hands a 16-byte raw record to the VALUE side (length bases, repcode history, packing, the store), which has no influence on
// the next state.  A lone warp spends about four cycles per instruction, so halving the chain warp's instructions halves the
// time of the longest frame.
struct SeqRaw { u32 v0, v1, a, b; };   // next 64 stream bits at the sequence start | LL cell with the offset's bit count in byte 1 | ML cell
struct SeqChain {
    u32 sLL, sOF, sML;
    int top;             // bit index of the next unread bit (drops below floorBit on overrun, then reads zeros)
    u32 k, nbSeq;

    template <class WS>
    ZB_HD void begin(WS& ws, u32 floorBit, u32 seqBits, u32 logLL, u32 logOF, u32 logML, u32 nbSeq_) {
        top = (int)(floorBit + seqBits) - 1;
        k = 0; nbSeq = nbSeq_;
        u32 W0, W1, W2, W3; ws.fetch4(top >> 5, W0, W1, W2, W3);
        u32 const c = 31u - ((u32)top & 31u);
        u32 const V0 = fshl32(W1, W0, c);
        u32 const t = logLL + logOF + logML;                 // <= 26
        u32 const y = shr_clamp(V0, 32 - t);
        sLL = y >> (logOF + logML); sOF = (y >> logML) & ((1u << logOF) - 1); sML = y & ((1u << logML) - 1);
        top -= (int)t;
        ws.advance(top >> 5);
    }
    // one sequence; `tLL/tOF/tML` = the frame's three tables (fse2 cells)
    // FAST: the caller guarantees that this is not the frame's last sequence and that the window lies above the stream's first
    // words (no masks); the bitstream request is predicated instead of branched -- a straight line for the warp.
    template <bool FAST, class WS>
    ZB_HD SeqRaw walk(WS& ws, const u32* tLL, const u32* tOF, const u32* tML) {
        u32 W0, W1, W2, W3;
        if (FAST) ws.fetch4_fast(top >> 5, W0, W1, W2, W3); else ws.fetch4(top >> 5, W0, W1, W2, W3);
        u32 const c = 31u - ((u32)top & 31u);
        u32 const V0 = fshl32(W1, W0, c), V1 = fshl32(W2, W1, c), V2 = fshl32(W3, W2, c);
        u32 const eLL = tLL[sLL], eOF = tOF[sOF], eML = tML[sML];
        u32 const S = eLL + eOF + eML;
        u32 const q2 = S & 0xFF, nTot = (S >> 8) & 0xFF;
        u32 const nOF = (eOF >> 8) & 0xFF, nML = (eML >> 8) & 0xFF;
        // read order: offset bits, ML extra, LL extra, then LL / ML / OF state bits (ZSTD_decodeSequence :1229-1346)
        bool const far = q2 >= 32;
        u32 const y = shr_clamp(fshl32(far ? V2 : V1, far ? V1 : V0, q2 & 31), 32 - nTot);
        bool const lastSeq = !FAST && (k + 1 == nbSeq);
        top -= (int)(q2 + (lastSeq ? 0u : nTot));
        if (FAST) ws.advance_fast(top >> 5); else ws.advance(top >> 5);      // the next step's four words are requested / waited for while this one finishes
        sLL = ((eLL >> 16) & 0x1FF) + (y >> (nML + nOF));
        sML = ((eML >> 16) & 0x1FF) + ((y >> nOF) & ((1u << nML) - 1));
        sOF = ((eOF >> 16) & 0x1FF) + (y & ((1u << nOF) - 1));
        ++k;
        SeqRaw r; r.v0 = V0; r.v1 = V1; r.a = (eLL & 0xFFFF00FFu) | ((eOF & 0xFF) << 8); r.b = eML;
        return r;
    }
    ZB_HD bool more() const { return k < nbSeq; }
    ZB_HD bool plain() const { return k + 1 < nbSeq && (top >> 5) >= 8; }      // walk<true>() may take the next sequence
    ZB_HD bool clean(u32 floorBit) const { return top + 1 == (int)floorBit; }       // every bit consumed, none borrowed
};
// The value side of one raw record: both lengths, the offset selector (idx 0..2 = repcode slot, 3 = rep0 - 1, 4 = a new offset) and
// the new offset the record would carry for idx 4.
struct SeqVal { u32 litLength, matchLength, idx, ofNew; };
ZB_HD SeqVal seq_value(SeqRaw const& r, const CodeTables* ct) {
    u32 const llBits = r.a & 0xFF, ofBits = (r.a >> 8) & 0xFF, mlBits = r.b & 0xFF;
    u32 const E = llBits + mlBits;
    u32 const ofVal = shr_clamp(r.v0, 32 - ofBits);
    u32 const x = shr_clamp(fshl32(r.v1, r.v0, ofBits & 31), 32 - E);
    u32 const llc = (r.a >> 25) & 0x3F, mlc = (r.b >> 25) & 0x3F;
    SeqVal s;
    s.litLength = ct->LL_base[llc < MaxLL ? llc : MaxLL] + (x & ((1u << (llBits & 31)) - 1));
    s.matchLength = ct->ML_base[mlc < MaxML ? mlc : MaxML] + (x >> (llBits & 31));
    u32 const ll0 = (llc == 0);          // :1300 tests litLength base == 0, true for code 0 only
    s.idx = ofBits > 1 ? 4u : ofBits + ll0 + ofVal;
    s.ofNew = ((1u << (ofBits & 31)) - 3) + ofVal;
    return s;
}
struct SeqValue {
    u32 rep0, rep1, rep2, k;
    u64* out;
    ZB_HD void begin(u64* out_) { rep0 = 1; rep1 = 4; rep2 = 8; k = 0; out = out_; }
    ZB_HD void take(SeqRaw const& r, const CodeTables* ct) { take_if(true, r, ct); }
    // `ok` false: the record was not there yet -- everything is computed, nothing is kept (selects instead of a branch: the value
    // warp polls 14 rings at once and must not diverge on which of them had news)
    ZB_HD void take_if(bool ok, SeqRaw const& r, const CodeTables* ct) {
        SeqVal const s = seq_value(r, ct);
        u32 const litLength = s.litLength, matchLength = s.matchLength, idx = s.idx;
        // offset / repcode history, all cases as selects: idx 0..3 = repcode slots (3: rep0 - 1), 4 = a new offset
        u32 cand = s.ofNew;                  // selects, not branches: lanes of a warp take all five cases at once
        cand = idx == 0 ? rep0 : cand; cand = idx == 1 ? rep1 : cand; cand = idx == 2 ? rep2 : cand; cand = idx == 3 ? rep0 - 1 : cand;
        cand -= !cand;                       // only a repcode can be zero here (rep0 - 1, or a corrupted history)
        u32 const n2 = idx >= 2 ? rep1 : rep2, n1 = idx >= 1 ? rep0 : rep1;
        rep2 = ok ? n2 : rep2; rep1 = ok ? n1 : rep1; rep0 = ok ? cand : rep0;
        u64 const l = umin(litLength, 0x3FFFFu), m = umin(matchLength, 0x3FFFFu), o = umin(cand, 0xFFFFFFFu);
        if (ok) out[k] = l | (m << 18) | (o << 36);
        k += ok ? 1u : 0u;
    }
};

// host / emulator form of stage C for one frame
ZB_HDN void dec_seq(DecDesc* d, const u8* blk, const u32* fse, const CodeTables* ct, u64* seqOut) {
    if (d->mode != 1 || d->stA1 || d->stA2 || d->nbSeq == 0 || d->seqUnusable) return;
    MemWords ws; ws.g.set(blk + d->seqOff);
    SeqChain D; SeqValue V;
    D.begin(ws, ws.g.floorBit, d->seqBits, d->logLL, d->logOF, d->logML, d->nbSeq);
    V.begin(seqOut);
    while (D.more()) {
        SeqRaw const r = D.plain() ? D.walk<true>(ws, fse, fse + FAST_FSE_OF, fse + FAST_FSE_ML) : D.walk<false>(ws, fse, fse + FAST_FSE_OF, fse + FAST_FSE_ML);
        V.take(r, ct);
    }
    if (!D.clean(ws.g.floorBit)) d->stC = E_corruption_detected;
}

// ---------------------------------------------------------------------------------------- stage B
// One thread per Huffman stream (HUF_decompress1X1_usingDTable_internal_body :574-595): the unread bits sit left
// aligned in a 64-bit register pair, the table index is a shift of its upper half, a 32-bit word slides in whenever 32
// bits or fewer are left.  step4() = four symbols and one aligned 32-bit store; step1() = one symbol (head / tail).
struct HufChain {
    u32 hi, lo;          // window, first unread bit on top of hi
    int avail;           // valid bits in the window
    int kNext;           // word that slides in next
    int budget;          // stream bits not yet moved into the window or consumed: ends at 0 exactly
    u32 left;            // symbols to go
    u8* op;

    template <class WS>
    ZB_HD void begin(WS& ws, u32 floorBit, u32 bits, u8* dst, u32 n) {
        int const top = (int)(floorBit + bits) - 1;
        int const k0 = top >> 5;
        u32 const c = 31u - ((u32)top & 31u);            // bits of word k0 above the end mark
        u32 const W0 = ws.word(k0), W1 = ws.word(k0 - 1);
        hi = fshl32(W1, W0, c); lo = W1 << c;            // whole words only: the low c bits stay empty until the next refill
        avail = 64 - (int)c; kNext = k0 - 2;
        budget = (int)bits;                              // consumed bits are counted against this
        left = n; op = dst;
    }
    template <class WS>
    ZB_HD void refill(WS& ws) {
        if (avail <= 32) {                               // 9 <= avail here: at most 2 x 12 bits leave between two refills
            u32 const wv = ws.word(kNext); kNext--;
            hi |= shr_clamp(wv, (u32)avail);             // avail == 32: nothing reaches hi
            lo = wv << (32u - (u32)avail);
            avail += 32;
            ws.advance(kNext);
        }
    }
    ZB_HD u32 symbol(const u16* table, u32 sh) {
        u32 const e = table[hi >> sh];
        u32 const nb = e >> 8;
        hi = fshl32(lo, hi, nb); lo <<= nb;              // nb <= 12
        avail -= (int)nb; budget -= (int)nb;
        return e & 0xFF;
    }
    template <class WS>
    ZB_HD void step4(WS& ws, const u16* table, u32 sh) {
        refill(ws); u32 const s0 = symbol(table, sh), s1 = symbol(table, sh);     // avail > 32 >= 2 x 12 bits
        refill(ws); u32 const s2 = symbol(table, sh), s3 = symbol(table, sh);
        *reinterpret_cast<u32*>(op) = s0 | (s1 << 8) | (s2 << 16) | (s3 << 24);
        op += 4; left -= 4;
    }
    // Straight-line form of refill() for the warp's common case (kNext above the stream's first words): the word is read
    // and the request for the next group issued whether needed or not, selects decide what sticks.
    template <class WS>
    ZB_HD void refill_fast(WS& ws) {
        bool const need = avail <= 32;
        u32 const wv = ws.raw(kNext);
        u32 const intoHi = shr_clamp(wv, (u32)avail), newLo = wv << ((32u - (u32)avail) & 31u);
        hi |= need ? intoHi : 0u; lo = need ? newLo : lo;
        avail += need ? 32 : 0; kNext -= need ? 1 : 0;
    }
    template <class WS>
    ZB_HD void step4_fast(WS& ws, const u16* table, u32 sh) {
        refill_fast(ws); u32 const s0 = symbol(table, sh), s1 = symbol(table, sh);
        refill_fast(ws); u32 const s2 = symbol(table, sh), s3 = symbol(table, sh);
        *reinterpret_cast<u32*>(op) = s0 | (s1 << 8) | (s2 << 16) | (s3 << 24);
        op += 4; left -= 4;
        ws.advance_fast(kNext);          // at most two words, i.e. one group, further down than before
    }
    ZB_HD bool plain() const { return left >= 8 && aligned4() && kNext >= 8; }      // step4_fast() may take the next four symbols
    template <class WS>
    ZB_HD void step1(WS& ws, const u16* table, u32 sh) {
        refill(ws); *op++ = (u8)symbol(table, sh); left--;
    }
    ZB_HD bool aligned4() const { return (reinterpret_cast<uintptr_t>(op) & 3) == 0; }
    ZB_HD bool clean() const { return budget == 0; }
};

// host / emulator form of stage B: stream k of one frame
ZB_HDN void dec_huf(DecDesc* d, int k, const u8* blk, const u16* huf, u8* lit) {
    if (d->mode != 1 || d->stA1 || d->litMode != 2 || k >= (int)d->nStreams || d->sBits[k] == NO_END_MARK) return;
    MemWords ws; ws.g.set(blk + d->sOff[k]);
    HufChain H;
    H.begin(ws, ws.g.floorBit, d->sBits[k], lit + d->oOff[k], d->oCnt[k]);
    u32 const sh = 32 - d->hufLog;
    while (H.left) { if (H.plain()) H.step4_fast(ws, huf, sh); else if (H.left >= 4 && H.aligned4()) H.step4(ws, huf, sh); else H.step1(ws, huf, sh); }
    if (!H.clean()) d->stB = E_corruption_detected;
}

// ---------------------------------------------------------------------------------------- stage D
// Warp per frame, "byte gather" (ZSTD_execSequence :1001-1096 without its ordering): groups of EXEC_G sequences get
// their output / literal positions by prefix sums and go to shared memory as 16-byte records; then the group's
// output span is produced 128 bytes per round, four consecutive bytes per lane.  A byte finds the sequence it
// belongs to through a small map of the sequence starts inside the round, and its source: a literal, or the byte
// `offset` back -- folded into the match's own history when the match overlaps itself (offset < position in
// match), and chased through the map while it still points into the round being written.  Everything before the
// round is final, so no lane ever waits for another.
constexpr u32 EXEC_SPL = 4;                  // sequences per lane and group
constexpr u32 EXEC_G = 32 * EXEC_SPL;      // on a 32-lane warp
struct alignas(16) ExecRec { u32 o, md, ls, off; };      // output start, match start (both counted from dst - A), literal start, offset
struct ExecShared {
    ExecRec rec[EXEC_G + 1];
    u32 st[EXEC_G + 1 + 64];     // rec[j].o again, then 0xFFFFFFFF: the sorted array the owner searches walk
    u32 tile[32];                // a round's bytes as far as they are known ...
    u32 late[32];                // ... which of them are not yet (bit t of word l: byte t of lane l) ...
    u32 link[32];                // ... and, for those, the byte of the round they copy (index inside the round, one byte each)
    u32 sum[2];                  // the frame's checksum: whether it has one, the stored 32 bits (dec_exec)
};
// Index (relative to `cur`) of the sequence that holds output position p: the last of st[cur .. cur+63] that is <= p.  A round of
// 128 bytes holds at most 43 sequence starts and st[cur] <= p for every byte that is looked up, so six halving steps decide.
ZB_HD u32 exec_owner(const u32* st, u32 p) {
    u32 u = 0;
    u += st[u + 32] <= p ? 32u : 0u; u += st[u + 16] <= p ? 16u : 0u; u += st[u + 8] <= p ? 8u : 0u;
    u += st[u + 4] <= p ? 4u : 0u; u += st[u + 2] <= p ? 2u : 0u; u += st[u + 1] <= p ? 1u : 0u;
    return u;
}

// a % b for a, b < 2^22 (positions inside a block): on the device through one reciprocal -- the quotient estimate is off by at most
// one, which two selects repair -- instead of the general 32-bit remainder; b == 0 (records beyond the group) yields garbage, never a trap
ZB_HD u32 exec_mod(u32 a, u32 b) {
#if defined(__CUDA_ARCH__)
    u32 const q = (u32)__float2uint_rz(__uint2float_rz(a) * __frcp_rz(__uint2float_rz(b)));
    u32 r = a - q * b;
    r = (int)r < 0 ? r + b : r;
    r = r >= b ? r - b : r;
    return r;
#else
    return b ? a % b : 0;
#endif
}

// The n bytes at dst a checksummed frame regenerated (written by the whole warp, which has synchronised since) against the stored 32 bits
// `want`: n, or checksum_wrong.  Not inlined: the hash's registers stay out of the executor's loop.
template <class C>
ZB_HDN size_t dec_checksum(const C& w, u32 want, const u8* dst, u32 n) {
    return (u32)xxh64_warp(w, dst, n) == want ? n : ERR(E_checksum_wrong);
}

template <class C>
ZB_HD size_t dec_exec_body(const C& w, ExecShared& X, const DecDesc* dp, const u8* item, const u8* litBuf, const u64* seqs, u8* dst, size_t cap) {
    DecDesc const& d = *dp;
    if (d.mode == 2 || d.mode == 3) {            // raw / rle block: 16-byte stores once dst is aligned
        u32 const n = d.mode == 2 ? d.cSize : d.regen;
        if (n > cap) return ERR(E_dstSize_tooSmall);
        const u8* const s = item + d.blockOff;
        u32 const v1 = d.rleByte * 0x01010101u;
        u32 head = (u32)((16 - (reinterpret_cast<uintptr_t>(dst) & 15)) & 15); if (head > n) head = n;
        for (u32 j = (u32)w.lane; j < head; j += C::W) dst[j] = d.mode == 2 ? s[j] : (u8)d.rleByte;
        u32 const body = (n - head) / 16;
        for (u32 j = (u32)w.lane; j < body; j += C::W) {
            u32 a0 = v1, a1 = v1, a2 = v1, a3 = v1;
            if (d.mode == 2) { u64 const lo = load64(s + head + 16 * j), hi = load64(s + head + 16 * j + 8); a0 = (u32)lo; a1 = (u32)(lo >> 32); a2 = (u32)hi; a3 = (u32)(hi >> 32); }
            u32* const t = reinterpret_cast<u32*>(dst + head + 16 * j);
#if defined(__CUDA_ARCH__)
            *reinterpret_cast<uint4*>(t) = make_uint4(a0, a1, a2, a3);
#else
            t[0] = a0; t[1] = a1; t[2] = a2; t[3] = a3;
#endif
        }
        for (u32 j = head + body * 16 + (u32)w.lane; j < n; j += C::W) dst[j] = d.mode == 2 ? s[j] : (u8)d.rleByte;
        w.sync();
        return n == d.contentSize ? n : ERR(E_corruption_detected);
    }
    // error precedence of the fused decoder: literals header/table, Huffman streams, sequences header/tables, then execution
    if (d.stA1) return ERR((int)d.stA1);
    if (d.stB) return ERR((int)d.stB);
    if (d.stA2) return ERR((int)d.stA2);
    if (d.nbSeq && cap == 0) return ERR(E_dstSize_tooSmall);
    if (cap > d.outMax) cap = d.outMax;
    if (d.nbSeq && d.seqUnusable) return ERR((int)d.stC);            // unusable stream: nothing was decoded
    const u8* const lit = d.litMode == 0 ? item + d.blockOff + d.rawOff : litBuf;
    bool const rle = d.litMode == 1; u32 const rleByte = d.rleByte;
    u32 const litSize = d.litSize, nbSeq = d.nbSeq;
    u32 const A = (u32)(reinterpret_cast<uintptr_t>(dst) & 3);      // rounds are aligned to 128 bytes of (dst - A)
    u8* const dstA = dst - A;
    constexpr u32 G = (u32)C::W * EXEC_SPL, ROUND = 4u * (u32)C::W;     // 128 sequences per group, 128 bytes per round on a 32-lane warp
    u32 op = 0, lp = 0;     // output / literal cursors (uniform)
    for (u32 base = 0; base < nbSeq; base += G) {
        // ---- the group's sequences: lane owns EXEC_SPL consecutive ones
        u32 ll[EXEC_SPL], ml[EXEC_SPL], off[EXEC_SPL];
        u32 sumO = 0, sumL = 0;
        for (u32 t = 0; t < EXEC_SPL; t++) {
            u32 const i = base + (u32)w.lane * EXEC_SPL + t;
            u64 const q = i < nbSeq ? seqs[i] : 0;
            ll[t] = (u32)(q & 0x3FFFF); ml[t] = (u32)((q >> 18) & 0x3FFFF); off[t] = (u32)(q >> 36);
            sumO += ll[t] + ml[t]; sumL += ll[t];
        }
        u32 o = op + w.exscan(sumO), ls = lp + w.exscan(sumL);
        // validity in sequence order (ZSTD_execSequenceEnd :919-932); `bad` = first failing sequence of the lane
        u32 code = 0, badAt = G;
        for (u32 t = 0; t < EXEC_SPL; t++) {
            u32 const i = base + (u32)w.lane * EXEC_SPL + t;
            u32 const md = o + ll[t];
            if (i < nbSeq && !code) {
                if ((size_t)ll[t] + ml[t] > cap - (size_t)(o < cap ? o : cap) || o > cap) code = E_dstSize_tooSmall;
                else if (ll[t] > litSize - (ls < litSize ? ls : litSize) || ls > litSize) code = E_corruption_detected;
                else if (off[t] > md) code = E_corruption_detected;
                if (code) badAt = (u32)w.lane * EXEC_SPL + t;
            }
            ExecRec r; r.o = o + A; r.md = md + A; r.ls = ls; r.off = off[t];
            X.rec[(u32)w.lane * EXEC_SPL + t] = r;
            X.st[(u32)w.lane * EXEC_SPL + t] = o + A;
            o = md + ml[t]; ls += ll[t];
        }
        u32 const badMask = w.ballot(code != 0);
        u32 nGood = nbSeq - base < G ? nbSeq - base : G;          // sequences of the group to execute
        u32 failCode = 0;
        if (badMask) { int const fl = (int)ctz32(badMask); nGood = w.shfl(badAt, fl); failCode = w.shfl(code, fl); }
        // end of the good prefix: start of sequence nGood (a sentinel record closes the table)
        u32 const endO = w.shfl(o, C::W - 1), endL = w.shfl(ls, C::W - 1);
        if (w.lane == 0 && nGood == G) { ExecRec r; r.o = endO + A; r.md = endO + A; r.ls = endL; r.off = 0; X.rec[G] = r; }
        if (w.lane == 0) X.st[G] = endO + A;
        if (badMask) for (u32 t = 0; t < EXEC_SPL; t++) { u32 const j = (u32)w.lane * EXEC_SPL + t; if (j > nGood) X.st[j] = 0xFFFFFFFFu; }      // positions after a bad sequence mean nothing: keep the array sorted
        for (u32 j = (u32)w.lane; j < 64; j += C::W) X.st[G + 1 + j] = 0xFFFFFFFFu;
        w.sync();
        u32 const gEndV = X.rec[nGood].o, gEnd = gEndV - A;          // for nGood < G that is a real record's start
        u32 const gEndL = X.rec[nGood].ls;
        // ---- rounds over [op, gEnd), in coordinates of (dst - A): v = position + A
        u32 const opV = op + A;
        u32 cur = 0;                              // first sequence that is not entirely before the round
        for (u32 rb = opV & ~(ROUND - 1); rb < gEndV; rb += ROUND) {
            u32 const floorV = rb > opV ? rb : opV;            // sources below this are final
            u32 const vb = rb + 4 * (u32)w.lane;               // the lane's first byte
            const u32* const st = X.st + cur;
            bool const single = st[1] >= rb + ROUND;           // no sequence starts inside the round after cur's own start
            // Long runs first: when this round and at least three more lie inside ONE literal run, or inside one match whose source
            // is far enough back (or repeats with a period of 1, 2 or 4 bytes), the bytes are moved as aligned words -- four per
            // lane and iteration, 512 bytes per warp iteration, each store instruction one contiguous 128-byte line -- without any
            // per-byte bookkeeping.  Everything shorter, nearer or odd goes through the rounds below.
            if (C::W == 32 && single && rb >= opV) {
                ExecRec const r = X.rec[cur];
                bool const inLit = rb + ROUND <= r.md, inMatch = rb >= r.md;
                u32 const segEnd = inLit ? r.md : (st[1] < gEndV ? st[1] : gEndV);
                u32 const span = (inLit || inMatch) && segEnd > rb ? ((segEnd - rb) & ~511u) : 0;
                bool const periodic = inMatch && (r.off == 1 || r.off == 2 || r.off == 4);
                if (span && (inLit ? true : (r.off >= 512 || periodic))) {
                    if ((inLit && rle) || periodic) {
                        u32 pat;
                        if (inLit) pat = rleByte * 0x01010101u;
                        else {      // the period starts at md - off; a 4-aligned v has the same phase everywhere because off divides 4
                            u32 const ph = (rb - r.md) & (r.off - 1);
                            pat = 0;
                            for (u32 j = 0; j < 4; j++) pat |= (u32)dstA[r.md - r.off + ((ph + j) & (r.off - 1))] << (8 * j);
                        }
                        for (u32 it = rb; it < rb + span; it += 512)
                            for (u32 j = 0; j < 4; j++) *reinterpret_cast<u32*>(dstA + it + 128 * j + 4 * (u32)w.lane) = pat;
                    } else {
                        const u8* const sb = inLit ? lit + (r.ls + (rb - r.o)) : dstA + (rb - r.off);      // source of byte rb
                        for (u32 it = rb; it < rb + span; it += 512) {
                            u32 wv[4];
                            for (u32 j = 0; j < 4; j++) {
                                const u8* const sp = sb + (it - rb) + 128 * j + 4 * (u32)w.lane;
                                uintptr_t const a = reinterpret_cast<uintptr_t>(sp);
                                u32 const sh = (u32)(a & 3) * 8;
                                const u32* const aw = reinterpret_cast<const u32*>(a & ~(uintptr_t)3);
                                u32 const w0 = aw[0], w1 = sh ? aw[1] : 0u;
                                wv[j] = fshr32(w0, w1, sh);
                            }
                            for (u32 j = 0; j < 4; j++) *reinterpret_cast<u32*>(dstA + it + 128 * j + 4 * (u32)w.lane) = wv[j];
                            if (!inLit) w.sync();               // a far match may still read what the previous iteration wrote
                        }
                    }
                    rb += span - ROUND;                         // (the loop adds the last ROUND)
                    w.sync();
                    continue;                                   // cur is unchanged: the run ended inside the same sequence
                }
            }
            bool const interior = rb >= opV && rb + ROUND <= gEndV;
            u32 u[4] = { 0, 0, 0, 0 };                          // per byte: index (relative to cur) of the sequence it belongs to
            if (!single) {
                u[0] = exec_owner(st, vb);
                u[1] = u[0] + (st[u[0] + 1] <= vb + 1 ? 1u : 0u);
                u[2] = u[1] + (st[u[1] + 1] <= vb + 2 ? 1u : 0u);
                u[3] = u[2] + (st[u[2] + 1] <= vb + 3 ? 1u : 0u);
            }
            u32 validMask = 15;
            if (!interior) { validMask = 0; for (u32 t = 0; t < 4; t++) if (vb + t >= opV && vb + t < gEndV) validMask |= 1u << t; }
            // first pass: where every byte comes from; a match folding onto itself reads from its first period.  Bytes whose source is
            // produced in this very round wait for the second pass.
            const u8* ad[4]; u32 srcV[4]; u32 lateMask = 0, litMask = 0;
            {   u32 rmd[4], roff[4], rlit[4]; u32 foldMask = 0;
                for (u32 t = 0; t < 4; t++) {
                    u32 const v = vb + t;
                    ExecRec const r = X.rec[cur + u[t]];
                    rmd[t] = r.md; roff[t] = r.off; rlit[t] = r.ls + (v - r.o);
                    u32 const sv = v - r.off;      // a match that overlaps itself may read `offset` back as long as that byte is final ...
                    srcV[t] = sv;
                    if (v < r.md) litMask |= 1u << t;
                    else if (sv >= floorV && v - r.md >= r.off) foldMask |= 1u << t;
                }
                if (w.ballot(foldMask != 0))       // ... if it is not, the match's first period holds the same byte
                    for (u32 t = 0; t < 4; t++) {
                        u32 const f = rmd[t] - roff[t] + exec_mod(vb + t - rmd[t], roff[t]);
                        srcV[t] = ((foldMask >> t) & 1) ? f : srcV[t];
                    }
                for (u32 t = 0; t < 4; t++) {
                    bool const isLit = (litMask >> t) & 1;
                    if (!isLit && srcV[t] >= floorV) lateMask |= 1u << t;
                    ad[t] = isLit ? lit + rlit[t] : dstA + srcV[t];
                } }
            lateMask &= validMask;
            u32 val;
            {   u32 const go = validMask & ~lateMask;
                u32 bt[4];
                for (u32 t = 0; t < 4; t++) bt[t] = ((go >> t) & 1) ? (u32)*ad[t] : 0u;
                if (rle) for (u32 t = 0; t < 4; t++) if ((litMask >> t) & 1) bt[t] = rleByte;
                val = bt[0] | (bt[1] << 8) | (bt[2] << 16) | (bt[3] << 24); }
            // second pass, only when some lane needs it: the round's bytes so far go to shared memory together with, for every byte that
            // is still missing, the index of the byte it copies.  A missing byte takes its source from there once that one is known;
            // until then it adopts its source's own link (pointer jumping: chains of copies inside a round -- up to 127 links for an
            // offset of one -- halve with every turn, so seven turns are the most a round can need)
            if (w.ballot(lateMask != 0)) {
                u32 lk = 0;
                for (u32 t = 0; t < 4; t++) lk |= ((srcV[t] - rb) & 0xFFu) << (8 * t);
                u32 pend = lateMask;
                X.tile[w.lane] = val; X.late[w.lane] = pend; X.link[w.lane] = lk;
                w.sync();
                for (;;) {
                    u32 nval = val, npend = pend, nlk = lk;
                    for (u32 t = 0; t < 4; t++) {               // straight line: the three words of every byte's source are fetched whether needed or not
                        u32 const j = (lk >> (8 * t)) & 0x7Fu, jw = j >> 2, js = 8 * (j & 3);
                        u32 const sLate = (X.late[jw] >> (j & 3)) & 1, sByte = (X.tile[jw] >> js) & 0xFFu, sLink = (X.link[jw] >> js) & 0xFFu;
                        bool const mine = (pend >> t) & 1, got = mine && !sLate, hop = mine && sLate;
                        nval |= got ? sByte << (8 * t) : 0u;
                        npend &= got ? ~(1u << t) : 0xFFFFFFFFu;
                        nlk = hop ? (nlk & ~(0xFFu << (8 * t))) | (sLink << (8 * t)) : nlk;
                    }
                    w.sync();                                   // every lane has read the turn's state
                    val = nval; pend = npend; lk = nlk;
                    X.tile[w.lane] = val; X.late[w.lane] = pend; X.link[w.lane] = lk;
                    if (!w.ballot(pend != 0)) break;
                    w.sync();
                }
            }
            if (validMask == 15) *reinterpret_cast<u32*>(dstA + vb) = val;
            else for (u32 t = 0; t < 4; t++) if ((validMask >> t) & 1) dstA[vb + t] = (u8)(val >> (8 * t));
            // the next round starts with the sequence holding this round's last byte, or the one after it if that one ends there
            u32 nc = cur + w.shfl(u[3], C::W - 1);
            if (nc < nGood && X.st[nc + 1] <= rb + ROUND) nc++;
            cur = nc < nGood ? nc : (nGood ? nGood - 1 : 0);
            w.sync();                                           // this round's bytes are sources of the next ones
        }
        if (failCode) return ERR((int)failCode);
        op = gEnd; lp = gEndL;
        w.sync();
    }
    if (nbSeq && d.stC) return ERR((int)d.stC);
    {   u32 const last = litSize - lp;
        if (last > cap - op) return ERR(E_dstSize_tooSmall);
        for (u32 k = (u32)w.lane; k < last; k += C::W) dst[op + k] = rle ? (u8)rleByte : lit[lp + k];
        op += last;
        w.sync(); }
    return op == d.contentSize ? op : ERR(E_corruption_detected);
}
// Stage D, then the frame's checksum when it has one (the flag in its descriptor byte, after the magic number unless magicless; the
// stored 32 bits right after its one block): the fused decoder's checks in its order -- content size (corruption_detected), then
// checksum_wrong.  The two go through shared memory (X.sum), so that nothing of the item stays live in registers across stage D.
template <class C>
ZB_HD size_t dec_exec(const C& w, ExecShared& X, const DecDesc* dp, const u8* item, const u8* litBuf, const u64* seqs, u8* dst, size_t cap,
                      u32 magicless = 0) {
    if (w.lane == 0) { u32 const has = (item[magicless ? 0 : 4] >> 2) & 1; X.sum[0] = has; X.sum[1] = has ? load32(item + dp->blockOff + dp->cSize) : 0u; }
    size_t const r = dec_exec_body(w, X, dp, item, litBuf, seqs, dst, cap);      // (a size comes back only after a warp synchronisation)
    if (isErr(r) || !X.sum[0]) return r;
    return dec_checksum(w, X.sum[1], dst, (u32)r);
}

}  // namespace zb
