// zb_decode_segment.cuh -- decoder for one frame of many blocks, a segment (a run of whole blocks) at a time, every stage parallel
// over the blocks of the segment or over its output bytes (kernels k_seg_* in zb_capi.cu):
//
//   A  seg_prepare  warp / block     prepare_block (zb_decode_fast.cuh): literal and sequence section headers, the tables the block
//                                    describes -> HBM, stream geometry
//   B  seg_tables   one thread       in block order: the earlier block (or the carried state) whose table a repeating block reuses
//   C  dec_huf      thread / stream  Huffman streams -> the block's literal buffer (zb_decode_fast.cuh)
//      seg_seq      thread / block   sequence stream -> lengths and raw offset selectors, and the block's repcode summary
//      seg_scan     one thread       output position of every block; the repcode history at every block start (summaries applied
//                                    in block order)
//      seg_offsets  thread / block   concrete offsets from the block's start history
//   D  seg_fill     warp / block     link map: every output byte of the segment is a final byte or the segment byte it copies
//      seg_jump     thread / byte    pointer jumping on the link map, in place, until every byte is final; the bytes -> dst
//
// Between segments the frame carries its output position, the repcode history and its last Huffman / FSE tables (SegCarry); nothing
// of it points into the input, so every segment may be read from its own staged copy.  Copies that reach before the segment read the
// history: the frame's output in dst (batch items, mask ~0), or a ring of a power-of-two size that keeps the last window of a streamed
// frame (zstdb200_fstream_*), at frame position & mask.
//
// seg_resume is the fused decoder entered at a block boundary: from the carried state and a linear copy of the history it decodes one
// segment's blocks and leaves the carried state as the segment decoder would, so the next segment may go either way.
//
// The segment path decides no error itself.  Whatever the fused decoder could reject -- a stage status, a table repeated before any
// block described it, a block regenerating more than blockSizeMax, an offset reaching before the frame, output beyond the capacity or
// the content size, a wrong checksum -- marks the frame `bad`, and the caller decodes it again on the fused kernel, whose bytes or
// error code are the result.  So valid frames decode to the same bytes and corrupted ones to the same error codes as before.
#pragma once
#include "zb_decode_fast.cuh"

namespace zb {

constexpr u32 SEG_HUF_ENTRIES = 1u << HUF_TABLELOG_MAX;
constexpr u32 SEG_CARRY = 0xFFFFFFFFu;       // table source: the state carried in from the frame's earlier segments
constexpr u32 SEG_NONE = 0xFFFFFFFEu;        // no table to reuse yet
constexpr u32 SEG_FINAL = 0x80000000u;       // link map entry: final byte in the low 8 bits; otherwise the index of the segment byte copied
constexpr u32 REP_LIT = 0xFFFFFFFFu;

// A repcode slot as a function of the history {in[0], in[1], in[2]} at the block's start: k == REP_LIT: the literal offset v; otherwise
// in[v] after k times `rep0 - 1` (ZSTD_decodeSequence :1300-1310: the result 0 becomes -1, `temp -= !temp`).  History values are never 0.
struct RepSym { u32 v, k; };
ZB_HD u32 rep_dec(u32 x, u32 k) { return x > k ? x - k : 0xFFFFFFFFu - (k - x); }
ZB_HD u32 rep_eval(RepSym s, const u32* in) { return s.k == REP_LIT ? s.v : rep_dec(in[s.v], s.k); }
// One sequence's offset selector: idx 0..2 = repcode slot, 3 = rep0 - 1, 4 = the new offset v.  Returns the offset taken.
ZB_HD u32 rep_step(u32* r, u32 idx, u32 v) {
    u32 const c = idx == 4 ? v : idx == 3 ? rep_dec(r[0], 1) : r[idx];
    if (idx >= 2) r[2] = r[1];
    if (idx >= 1) r[1] = r[0];
    r[0] = c;
    return c;
}
ZB_HD void rep_step_sym(RepSym* r, u32 idx, u32 v) {
    RepSym c = r[idx < 3 ? idx : 0];
    if (idx == 4) { c.v = v; c.k = REP_LIT; }
    else if (idx == 3) { if (c.k == REP_LIT) c.v = rep_dec(c.v, 1); else c.k += 1; }
    if (idx >= 2) r[2] = r[1];
    if (idx >= 1) r[1] = r[0];
    r[0] = c;
}

struct SegBlock {
    DecDesc d;           // as in the staged decoder; blockOff relative to the frame, mode 1 compressed / 2 raw / 3 rle
    u32 litType;         // literals block type of a compressed block (3: the previous Huffman table again)
    u32 fseRepeat;       // bit t: FSE table t (LL, OF, ML) is the previous one again
    u32 hufSrc, fseSrc[3];    // segment block whose table the block uses, or SEG_CARRY
    u32 bad;             // the frame goes to the fused decoder
    u32 regen;
    u64 out;             // item position of the block's first output byte (a frame of its own: frame position)
    u64 frameAt, segAt;  // item positions of its frame's first output byte and of its item's first output byte in the segment
    u32 linkAt;          // link map entry of the byte at segAt
    u64 sumLL, sumML;
    u32 rep[3];          // repcode history at the block's start
    RepSym sum[3];       // ... and at its end, as functions of rep
};

struct SegCarry {
    u64 pos, cap;        // output bytes of the item so far, output capacity of the item
    u64 frameAt;         // item position where the frame in progress starts
    u32 bad;
    u32 links;           // link map entries of the segment just scanned
    u32 hasHuf, hufLog, hasFse, fseLog[3];
    u32 rep[3];
    u32 nextHuf, nextFse[3];  // the last describing blocks of the segment just prepared (SEG_CARRY / SEG_NONE: none there)
    u16 huf[SEG_HUF_ENTRIES];
    u32 fse[FAST_FSE_ENTRIES];
};

// The largest window the segment decoder takes (the default windowLogMax): larger ones stay with the fused decoder.
constexpr u64 SEG_WINDOW_MAX = 1ull << 27;

// Host side: the blocks of an item the segment decoder takes, one frame (frame_walk, in the format `magicless` names) of more than one
// block with a window of at most SEG_WINDOW_MAX.  Returns the number of blocks, 0 for any other item.
ZB_HDN u32 seg_walk(const u8* src, size_t size, FrameHeader* fh, u64* refs, u32* xxh, u32 magicless = 0) {
    u32 const n = frame_walk(src, size, fh, 0xFFFFFFFFu, refs, xxh, nullptr, magicless);
    return n >= 2 && fh->windowSize <= SEG_WINDOW_MAX ? n : 0;
}

// ---------------------------------------------------------------------------------------- the device call's loop
// zstdb200_decompress_device plans on the GPU: each item is walked there (seg_item_blocks), and the blocks of all the items the loop takes
// form one sequence, cut into segments of B blocks that may cross frame and item boundaries.  A block carries its place in it (SegLoc);
// at a frame start the stages drop the earlier tables and restart the repcodes, at an item start the output position.  Any doubt marks
// the whole item in `itemBad`, and the fused decoder decodes it again; the loop decides no error.

// The blocks of an item the loop takes: a whole number of frames -- zstd frames (frame_walk) with a window of at most SEG_WINDOW_MAX,
// skippable ones unless magicless -- at least one zstd frame, and a frame of two blocks or two frames.  0 for any other item.
ZB_HDN u64 seg_item_blocks(const u8* src, size_t size, u32 magicless) {
    if (size > 0xFFFFFFFFu) return 0;
    size_t pos = 0; u64 blocks = 0; u32 frames = 0, zframes = 0, most = 0;
    while (pos < size) {
        size_t const rest = size - pos;
        if (!magicless && rest >= 8 && (load32(src + pos) & 0xFFFFFFF0u) == 0x184D2A50u) {
            if ((u64)load32(src + pos + 4) + 8 > rest) return 0;
            pos += 8 + (size_t)load32(src + pos + 4);
        } else {
            FrameHeader fh; size_t end = 0; u32 xxh;
            u32 const nb = frame_walk(src + pos, rest, &fh, 0xFFFFFFFFu, nullptr, &xxh, &end, magicless);
            if (!nb || fh.windowSize > SEG_WINDOW_MAX) return 0;
            blocks += nb; zframes++; most = nb > most ? nb : most; pos += end;
        }
        frames++;
    }
    return zframes && (most >= 2 || frames >= 2) ? blocks : 0;
}

// A block of the loop: its item, its frame's blockSizeMax, and flags -- it starts its item, starts its frame, ends its frame (then with
// the frame's stored checksum and declared content size when it has them); cap: the item's output capacity.
struct SegLoc { u32 item, flags, blockSizeMax, xxh; u64 cap, contentSize; };
constexpr u32 LOC_ITEM = 1, LOC_FRAME = 2, LOC_END = 4, LOC_CHECKSUM = 8, LOC_SIZE = 16;

// Which candidates go to the loop.  The loop decodes its blocks one segment after another, at about the same rate whatever their items;
// the fused kernel decodes `warps` items at once, each with one warp that is about SEG_FUSED_BLOCK_COST times slower per block than the
// loop (H100, level-3 frames: 0.011 GB/s per warp against 2.1 GB/s for the loop).  So a few long items belong on the loop and many short
// ones on the fused kernel.  The candidates are counted in buckets of floor(log2(blocks)) -- cnt, sum and max of the block counts -- and
// the least number of blocks an item needs to go to the loop is the power of two with the least estimated time of the fused kernel
// (the longer of its longest item and its blocks spread over the warps) plus the loop (its blocks); ~0 sends every item to the fused kernel.
constexpr u32 SEG_BUCKETS = 33;
constexpr u64 SEG_FUSED_BLOCK_COST = 200;
ZB_HDN u64 seg_loop_min_blocks(const u32* cnt, const u64* sum, const u32* max, u64 warps) {
    u64 loop = 0;
    for (u32 k = 0; k < SEG_BUCKETS; k++) loop += sum[k];
    u64 best = ~0ull, bestCost = ~0ull, fusedSum = 0, fusedMax = 0;
    for (u32 k = 0; k <= SEG_BUCKETS; k++) {      // items of fewer than 2^k blocks fused, the others on the loop
        u64 const spread = (fusedSum + warps - 1) / warps, fused = (fusedMax > spread ? fusedMax : spread) * SEG_FUSED_BLOCK_COST;
        if (fused + loop < bestCost) { bestCost = fused + loop; best = k < SEG_BUCKETS ? 1ull << k : ~0ull; }
        if (k < SEG_BUCKETS) { fusedSum += sum[k]; loop -= sum[k]; if (cnt[k] && max[k] > fusedMax) fusedMax = max[k]; }
    }
    return best;
}
// The bucket of an item of b >= 1 blocks.
ZB_HD u32 seg_bucket(u64 b) { u32 k = 0; while (k + 1 < SEG_BUCKETS && (b >> (k + 1))) k++; return k; }

// The loop's cursor: the call's items (list[0 .. count): the loop's, in the order walked) and the walk's position among their blocks.
struct SegCursor {
    const u8* src; const u64* srcOff; u8* dst; const u64* dstOff; u64* results;
    u32* itemBad;                // per item of the call: nonzero when the fused decoder decodes it again
    u32* list; u32 count, magicless;
    u32 k, at, inFrame, first;   // list index, byte offset in its item, 1 inside a frame (2: before its first block), next block starts the item
    u32 blockSizeMax, checksum, hasSize; u64 contentSize;      // the frame walked
    u32 n;                       // blocks in the segment walked last
    u32 cnt[SEG_BUCKETS], max[SEG_BUCKETS]; u64 sum[SEG_BUCKETS];      // the candidates (seg_loop_min_blocks)
    u64 minBlocks;               // the least blocks of an item on the loop
};

// Walks the next segment: up to B blocks from the cursor into refs (offset in the item | header << 32) and loc; returns their number.
// The items were walked whole before (seg_item_blocks), so every header read here is inside its item.
ZB_HDN u32 seg_walk_segment(SegCursor* c, u32 B, u64* refs, SegLoc* loc) {
    u32 n = 0;
    while (n < B && c->k < c->count) {
        u32 const item = c->list[c->k];
        const u8* const src = c->src + c->srcOff[item];
        u32 const size = (u32)(c->srcOff[item + 1] - c->srcOff[item]);
        if (!c->inFrame) {
            if (c->at == size) { c->k++; c->at = 0; c->first = 1; continue; }
            if (!c->magicless && size - c->at >= 8 && (load32(src + c->at) & 0xFFFFFFF0u) == 0x184D2A50u) { c->at += 8 + load32(src + c->at + 4); continue; }
            FrameHeader fh;
            read_frame_header(&fh, src + c->at, size - c->at, c->magicless);
            c->blockSizeMax = fh.blockSizeMax; c->checksum = fh.checksum; c->hasSize = fh.hasContentSize; c->contentSize = fh.contentSize;
            c->at += fh.headerSize; c->inFrame = 2;
        }
        u32 const bh = load24(src + c->at), cSize = ((bh >> 1) & 3) == 1 ? 1 : bh >> 3;
        SegLoc L;
        L.item = item; L.blockSizeMax = c->blockSizeMax; L.xxh = 0; L.cap = c->dstOff[item + 1] - c->dstOff[item]; L.contentSize = c->contentSize;
        L.flags = (c->first ? LOC_ITEM : 0u) | (c->inFrame == 2 ? LOC_FRAME : 0u);
        refs[n] = (u64)c->at | ((u64)bh << 32);
        c->at += 3 + cSize; c->first = 0; c->inFrame = 1;
        if (bh & 1) {
            L.flags |= LOC_END | (c->checksum ? LOC_CHECKSUM : 0u) | (c->hasSize ? LOC_SIZE : 0u);
            if (c->checksum) { L.xxh = load32(src + c->at); c->at += 4; }
            c->inFrame = 0;
        }
        loc[n++] = L;
    }
    c->n = n;
    return n;
}

// ---------------------------------------------------------------------------------------- stage A
// `bh` = the block header, at frame + off.  The fused decoder takes the frame when a block is refused or has a nonzero stage status.
template <class C>
ZB_HDN void seg_prepare(const C& w, DecShared& S, const u8* frame, u32 off, u32 bh, u32 blockSizeMax, SegBlock* b, u16* hufOut, u32* fseOut) {
    SegBlock B;
    memset(&B, 0, sizeof B);
    DecDesc& L = B.d;
    L.outMax = 0xFFFFFFFFu;
    if (w.lane == 0) { S.litEntropy = 1; S.fseEntropy = 1; }      // repeats are resolved by seg_tables
    w.sync();
    bool const ok = prepare_block(w, S, frame, off, bh, blockSizeMax, blockSizeMax, HUF_TABLELOG_MAX, L, hufOut, fseOut);
    B.bad = !ok || L.stA1 || L.stB || L.stA2 || L.stC;
    if (!B.bad && L.mode == 1) {
        B.litType = frame[off + 3] & 3;
        for (int t = 0; t < 3 && L.nbSeq; t++) B.fseRepeat |= (S.fseMode[t] == 3 ? 1u : 0u) << t;
    }
    w.sync();
    if (w.lane == 0) *b = B;
    w.sync();
}

// ---------------------------------------------------------------------------------------- stage B
// In block order: the table every repeating block reuses (ZSTD_decodeLiteralsBlock :148 / ZSTD_buildSeqTable :686).  The first
// segment of a frame starts the carried state.
// In the loop (loc, itemBad): at a frame start no earlier table; a failing block marks its item and the walk goes on with the next one.
ZB_HDN void seg_tables(SegBlock* blocks, u32 n, SegCarry* c, bool first, u64 cap, const SegLoc* loc = nullptr, u32* itemBad = nullptr) {
    if (first) {
        c->pos = 0; c->cap = cap; c->bad = 0; c->hasHuf = 0; c->hasFse = 0; c->frameAt = 0;
        c->rep[0] = 1; c->rep[1] = 4; c->rep[2] = 8;
    }
    u32 huf = c->hasHuf ? SEG_CARRY : SEG_NONE, fse[3];
    for (int t = 0; t < 3; t++) fse[t] = c->hasFse ? SEG_CARRY : SEG_NONE;
    for (u32 j = 0; j < n && !c->bad; j++) {
        SegBlock& B = blocks[j];
        u32* const bad = loc ? itemBad + loc[j].item : &c->bad;
        if (loc && (loc[j].flags & LOC_FRAME)) {
            huf = SEG_NONE; c->hasHuf = 0; c->hasFse = 0;
            for (int t = 0; t < 3; t++) fse[t] = SEG_NONE;
        }
        if (*bad) continue;
        if (B.bad) { *bad = 1; continue; }
        if (B.d.mode != 1) continue;
        if (B.litType == 3) {
            if (huf == SEG_NONE) { *bad = 1; continue; }
            B.hufSrc = huf; B.d.hufLog = huf == SEG_CARRY ? c->hufLog : blocks[huf].d.hufLog;
        } else if (B.litType == 2) huf = j;
        if (B.d.nbSeq) {
            for (int t = 0; t < 3; t++) {
                if ((B.fseRepeat >> t) & 1) {
                    if (fse[t] == SEG_NONE) { *bad = 1; break; }
                    B.d.fseLog[t] = fse[t] == SEG_CARRY ? c->fseLog[t] : blocks[fse[t]].d.fseLog[t];
                } else fse[t] = j;
                B.fseSrc[t] = fse[t];
            }
        }
    }
    c->nextHuf = huf;
    for (int t = 0; t < 3; t++) c->nextFse[t] = fse[t];
}

// ---------------------------------------------------------------------------------------- stage C
// Huffman stream k of block j, with the table the block uses.
ZB_HDN void seg_huf(SegBlock* blocks, u32 j, int k, const u8* frame, const u16* hufBase, const SegCarry* c, u8* lit) {
    SegBlock& B = blocks[j];
    u32 const src = B.litType == 3 ? B.hufSrc : j;
    dec_huf(&B.d, k, frame + B.d.blockOff, src == SEG_CARRY ? c->huf : hufBase + (size_t)src * SEG_HUF_ENTRIES, lit);
}

// Block j's sequence stream: lengths | selector << 36 to seqs, the new offset of a selector 4 to offs; the summary of its repcodes.
ZB_HDN void seg_seq(SegBlock* blocks, u32 j, const u8* frame, const u32* fseBase, const SegCarry* c, u64* seqs, u32* offs) {
    SegBlock& B = blocks[j];
    for (u32 s = 0; s < 3; s++) { B.sum[s].v = s; B.sum[s].k = 0; }
    B.sumLL = 0; B.sumML = 0;
    if (B.d.mode != 1 || B.d.nbSeq == 0) return;
    const u32* t[3];
    for (int k = 0; k < 3; k++) t[k] = (B.fseSrc[k] == SEG_CARRY ? c->fse : fseBase + (size_t)B.fseSrc[k] * FAST_FSE_ENTRIES) + fse_at(k);
    MemWords ws; ws.g.set(frame + B.d.blockOff + B.d.seqOff);
    SeqChain D;
    D.begin(ws, ws.g.floorBit, B.d.seqBits, B.d.logLL, B.d.logOF, B.d.logML, B.d.nbSeq);
    RepSym sum[3] = { { 0, 0 }, { 1, 0 }, { 2, 0 } };
    u64 sLL = 0, sML = 0;
    const CodeTables* const ct = &ZB_T;
    for (u32 k = 0; D.more(); k++) {
        SeqRaw const r = D.plain() ? D.walk<true>(ws, t[0], t[1], t[2]) : D.walk<false>(ws, t[0], t[1], t[2]);
        SeqVal const s = seq_value(r, ct);          // the offset stays a selector until the block's start history is known
        u64 const l = umin(s.litLength, 0x3FFFFu), m = umin(s.matchLength, 0x3FFFFu);
        seqs[k] = l | (m << 18) | ((u64)s.idx << 36);
        offs[k] = s.ofNew;
        rep_step_sym(sum, s.idx, s.ofNew);
        sLL += l; sML += m;
    }
    if (!D.clean(ws.g.floorBit)) B.bad = 1;
    for (int s = 0; s < 3; s++) B.sum[s] = sum[s];
    B.sumLL = sLL; B.sumML = sML;
}

// Output positions and start histories, in block order (after stage C).  Every block gets its item position (out), its frame's (frameAt)
// and its place in the link map: the item's bytes of the segment from segAt on are the entries from linkAt on.  In the loop a block
// starting an item starts its position at 0 and its capacity at loc's, a block starting a frame restarts the repcodes there.
ZB_HDN void seg_scan(SegBlock* blocks, u32 n, SegCarry* c, u32 blockSizeMax, const SegLoc* loc = nullptr, u32* itemBad = nullptr) {
    if (c->bad) return;
    u64 pos = c->pos, cap = c->cap, frameAt = c->frameAt, segAt = pos;
    u32 rep[3] = { c->rep[0], c->rep[1], c->rep[2] }, links = 0, linkAt = 0;
    for (u32 j = 0; j < n; j++) {
        SegBlock& B = blocks[j];
        u32* bad = &c->bad; u32 bsm = blockSizeMax;
        if (loc) {
            SegLoc const& L = loc[j];
            bad = itemBad + L.item; bsm = L.blockSizeMax;
            if (L.flags & LOC_ITEM) { pos = 0; cap = L.cap; segAt = 0; linkAt = links; }
            if (L.flags & LOC_FRAME) { frameAt = pos; rep[0] = 1; rep[1] = 4; rep[2] = 8; }
        }
        B.out = pos; B.frameAt = frameAt; B.segAt = segAt; B.linkAt = linkAt; B.regen = 0;
        if (*bad) continue;
        u64 regen = B.d.regen;
        if (B.d.mode == 1) {
            if (B.bad || B.d.stB || B.d.stC || B.sumLL > B.d.litSize) { *bad = 1; if (loc) continue; return; }
            regen = B.d.litSize + B.sumML;
        }
        if (regen > bsm || regen > cap - pos) { *bad = 1; if (loc) continue; return; }
        B.regen = (u32)regen; pos += regen; links += (u32)regen;
        for (int s = 0; s < 3; s++) B.rep[s] = rep[s];
        if (B.d.mode == 1 && B.d.nbSeq) {
            u32 nr[3];
            for (int s = 0; s < 3; s++) nr[s] = rep_eval(B.sum[s], rep);
            for (int s = 0; s < 3; s++) rep[s] = nr[s];
        }
    }
    c->pos = pos; c->cap = cap; c->frameAt = frameAt; c->links = links;
    for (int s = 0; s < 3; s++) c->rep[s] = rep[s];
}

// Block j: concrete offsets from its start history, in place over the new offsets.
ZB_HDN void seg_offsets(const SegBlock* blocks, u32 j, const u64* seqs, u32* offs) {
    SegBlock const& B = blocks[j];
    if (B.d.mode != 1) return;
    u32 r[3] = { B.rep[0], B.rep[1], B.rep[2] };
    for (u32 k = 0; k < B.d.nbSeq; k++) offs[k] = rep_step(r, (u32)(seqs[k] >> 36), offs[k]);
}

// The tables the next segment may reuse, into the carried state (after stage C read the old ones).
template <class C>
ZB_HD void seg_carry_tables(const C& w, const SegBlock* blocks, const u16* hufBase, const u32* fseBase, SegCarry* c) {
    if (c->bad) return;
    if (c->nextHuf < SEG_NONE) {
        u32 const j = c->nextHuf;
        for (u32 i = (u32)w.lane; i < SEG_HUF_ENTRIES; i += C::W) c->huf[i] = hufBase[(size_t)j * SEG_HUF_ENTRIES + i];
        if (w.lane == 0) { c->hufLog = blocks[j].d.hufLog; c->hasHuf = 1; }
    }
    for (int t = 0; t < 3; t++) {
        if (c->nextFse[t] >= SEG_NONE) continue;
        u32 const j = c->nextFse[t];
        for (u32 i = fse_at(t) + (u32)w.lane; i < fse_at(t + 1); i += C::W) c->fse[i] = fseBase[(size_t)j * FAST_FSE_ENTRIES + i];
        if (w.lane == 0) { c->fseLog[t] = blocks[j].d.fseLog[t]; c->hasFse = 1; }
    }
    w.sync();
}

// ---------------------------------------------------------------------------------------- stage D
// Block j's bytes into the segment's link map (entry linkAt + p - segAt for item position p): literal bytes and bytes copied from before
// the segment are final, a match byte inside the segment names the entry it copies -- for a match that overlaps itself, the byte of its
// first period, so that a run is one link deep.  Sequences go 32 at a time, their bytes are spread over the lanes.
struct SegRec { u64 o, md; u32 ls, off; };
// `hist`: the item's output before the segment, item position p at hist[p & mask]; an offset before the frame or beyond `window` sets
// *bad.
template <class C>
ZB_HDN void seg_fill(const C& w, SegRec* R, const SegBlock* blocks, u32 j, const u8* frame, const u8* lit, const u64* seqs, const u32* offs,
                     const u8* hist, u64 mask, u64 window, u32* link, u32* bad) {
    SegBlock const& B = blocks[j];
    u64 const base = B.out;
    auto put = [&](u64 p, u32 v) { link[B.linkAt + (p - B.segAt)] = v; };
    if (B.d.mode == 2 || B.d.mode == 3) {
        const u8* const s = frame + B.d.blockOff;
        for (u32 i = (u32)w.lane; i < B.regen; i += C::W) put(base + i, SEG_FINAL | (B.d.mode == 2 ? s[i] : B.d.rleByte));
        w.sync();
        return;
    }
    const u8* const L = B.d.litMode == 0 ? frame + B.d.blockOff + B.d.rawOff : lit;
    bool const rle = B.d.litMode == 1;
    u64 op = base; u32 lp = 0;
    for (u32 s0 = 0; s0 < B.d.nbSeq; s0 += C::W) {
        u32 const i = s0 + (u32)w.lane;
        u64 const q = i < B.d.nbSeq ? seqs[i] : 0;
        u32 const ll = (u32)(q & 0x3FFFF), ml = (u32)((q >> 18) & 0x3FFFF), off = i < B.d.nbSeq ? offs[i] : 0;
        u64 const o = op + w.exscan(ll + ml);
        u32 const ls = lp + w.exscan(ll);
        bool const far = i < B.d.nbSeq && ((u64)off > o + ll - B.frameAt || off > window);     // before the frame (ZSTD_execSequence :1034) or the window
        if (w.ballot(far)) { if (w.lane == 0) *bad = 1; return; }
        SegRec r; r.o = o; r.md = o + ll; r.ls = ls; r.off = off;
        R[w.lane] = r;
        u32 const cnt = B.d.nbSeq - s0 < (u32)C::W ? B.d.nbSeq - s0 : (u32)C::W;
        u64 const end = w.shfl(o + ll + ml, (int)cnt - 1);
        u32 const lend = w.shfl(ls + ll, (int)cnt - 1);
        w.sync();
        u32 u = 0;
        for (u64 p = op + (u32)w.lane; p < end; p += C::W) {
            while (u + 1 < cnt && R[u + 1].o <= p) u++;       // bytes of a lane only move forward
            SegRec const& e = R[u];
            u32 v;
            if (p < e.md) v = SEG_FINAL | (rle ? B.d.rleByte : L[e.ls + (u32)(p - e.o)]);
            else {
                u64 const src = e.md - e.off + (p - e.md) % e.off;
                v = src < B.segAt ? SEG_FINAL | hist[src & mask] : B.linkAt + (u32)(src - B.segAt);
            }
            put(p, v);
        }
        w.sync();
        op = end; lp = lend;
    }
    for (u32 k = (u32)w.lane; k < B.d.litSize - lp; k += C::W) put(op + k, SEG_FINAL | (rle ? B.d.rleByte : L[lp + k]));
    w.sync();
}

// One frame a segment at a time (segStart: blocks[0].out, which the blocks carry as segAt): the history at hist[p & mask], or the frame's
// whole output in dst.
template <class C>
ZB_HDN void seg_fill(const C& w, SegRec* R, const SegBlock* blocks, u32 j, const u8* frame, const u8* lit, const u64* seqs, const u32* offs,
                     const u8* hist, u64 mask, u64 window, u64 segStart, u32* link, SegCarry* c) {
    (void)segStart;
    seg_fill(w, R, blocks, j, frame, lit, seqs, offs, hist, mask, window, link, &c->bad);
}
template <class C>
ZB_HDN void seg_fill(const C& w, SegRec* R, const SegBlock* blocks, u32 j, const u8* frame, const u8* lit, const u64* seqs, const u32* offs,
                     const u8* dst, u64 segStart, u32* link, SegCarry* c) {
    seg_fill(w, R, blocks, j, frame, lit, seqs, offs, dst, ~0ull, ~0ull, segStart, link, c);
}

// Segment byte p: follows its links, shortening its own entry on the way (others that reach it later jump further), until a final
// byte.  Every link points to an earlier byte, so the walk ends; an entry only ever changes to another entry on its own chain.
ZB_HD u8 seg_jump(volatile u32* link, u32 p) {
    u32 v = link[p];
    while (!(v & SEG_FINAL)) { v = link[v]; link[p] = v; }
    return (u8)v;
}


// The loop's frame that ends with block j (LOC_END), its item not marked: its declared content size, and its checksum over its output
// dst[frameAt, end) with the whole warp.  Either wrong marks the item.  Returns the item position where the frame ends.
template <class C>
ZB_HDN u64 seg_frame_end(const C& w, const SegBlock* blocks, u32 j, const SegLoc& L, const u8* dst, u32* bad) {
    SegBlock const& B = blocks[j];
    u64 const end = B.out + B.regen, len = end - B.frameAt;
    bool ok = !(L.flags & LOC_SIZE) || len == L.contentSize;
    if (ok && (L.flags & LOC_CHECKSUM)) ok = (u32)xxh64_warp(w, dst + B.frameAt, (size_t)len) == L.xxh;
    if (!ok && w.lane == 0) *bad = 1;
    return end;
}

// ---------------------------------------------------------------------------------------- resume
// The fused decoder (zb_decode.cuh) from a block boundary: the n blocks at in + (u32)refs[j] (headers refs[j] >> 32) of the segment that
// starts at frame position c->pos, written to out, with the history hist[0, out - hist) right before it -- offsets reaching before
// hist are corruption, as they are before the frame start.  The repcodes and the last tables come from the carried state and go back
// to it; the FSE cells are carried in the staged format (fse2_pack), which keeps the fields of the fused format.  Returns the bytes
// written or the fused decoder's error code.
ZB_HD u32 fse2_unpack(u32 e) { return ((e >> 16) & 0x1FFu) | (((e >> 8) & 0xFFu) << 16) | ((e >> 25) << 24); }
template <class C>
ZB_HDN size_t seg_resume(const C& w, DecShared& S, const u8* in, const u64* refs, u32 n, u32 blockSizeMax, const u8* hist, u8* out,
                         size_t cap, u8* scratch, SegCarry* c) {
    if (w.lane == 0) {
        for (int s = 0; s < 3; s++) { S.rep[s] = c->rep[s]; S.fseLog[s] = c->fseLog[s]; }
        S.litEntropy = c->hasHuf; S.fseEntropy = c->hasFse; S.hufLog = c->hufLog;
    }
    w.sync();
    if (c->hasHuf) for (u32 i = (u32)w.lane; i < (1u << c->hufLog); i += C::W) S.huf[i] = c->huf[i];
    if (c->hasFse)
        for (int t = 0; t < 3; t++)
            for (u32 i = (u32)w.lane; i < (1u << c->fseLog[t]); i += C::W) S.fse[t][i] = fse2_unpack(c->fse[fse_at(t) + i]);
    w.sync();
    size_t written = 0;
    for (u32 j = 0; j < n; j++) {
        u32 const bh = (u32)(refs[j] >> 32), type = (bh >> 1) & 3;
        size_t const cSize = type == 1 ? 1 : bh >> 3;
        const u8* const ip = in + (u32)refs[j] + 3;
        size_t decoded;
        if (type == 2) {
            decoded = decode_block(w, S, hist, out + written, cap - written, ip, cSize, blockSizeMax, scratch);
            if (isErr(decoded)) return decoded;
        } else if (type == 0) {
            if (cSize > cap - written) return ERR(E_dstSize_tooSmall);
            for (size_t k = (size_t)w.lane; k < cSize; k += C::W) out[written + k] = ip[k];
            decoded = cSize; w.sync();
        } else if (type == 1) {
            size_t const rl = bh >> 3;
            if (rl > cap - written) return ERR(E_dstSize_tooSmall);
            for (size_t k = (size_t)w.lane; k < rl; k += C::W) out[written + k] = ip[0];
            decoded = rl; w.sync();
        } else return ERR(E_corruption_detected);
        written += decoded;
    }
    if (S.litEntropy) for (u32 i = (u32)w.lane; i < (1u << S.hufLog); i += C::W) c->huf[i] = S.huf[i];
    if (S.fseEntropy)
        for (int t = 0; t < 3; t++)
            for (u32 i = (u32)w.lane; i < (1u << S.fseLog[t]); i += C::W) {
                u32 const e = S.fse[t][i], sym = e >> 24;
                c->fse[fse_at(t) + i] = fse2_pack(e, t == 0 ? ZB_T.LL_bits[sym] : t == 1 ? sym : ZB_T.ML_bits[sym]);
            }
    w.sync();
    if (w.lane == 0) {
        for (int s = 0; s < 3; s++) { c->rep[s] = S.rep[s]; c->fseLog[s] = S.fseLog[s]; }
        c->hasHuf = S.litEntropy; c->hasFse = S.fseEntropy; c->hufLog = S.hufLog; c->pos += written;
    }
    w.sync();
    return written;
}

// A streamed frame's block the reference's streaming decoder rejects from its 3-byte header `bh` alone: a reserved type, or more than
// blockSizeMax bytes of block content or of RLE output (ZSTD_decompressContinue, corruption_detected).
ZB_HD bool stream_block_error(u32 bh, u32 blockSizeMax) {
    return ((bh >> 1) & 3) == 3 || (bh >> 3) > blockSizeMax;
}

// The frame stream's result of a segment on the resume entry.  The fused decoder stops a damaged block at blockSizeMax + 32 bytes of
// output with dstSize_tooSmall, as the reference's one-shot decoder does; the reference's streaming decoder decodes into a buffer with
// room beyond the block and rejects the block at its end with corruption_detected (ZSTD_decompressContinue :1367).  With the resume
// entry's room, dstSize_tooSmall can only be that limit, so the stream reports the streaming decoder's code.
ZB_HD size_t stream_resume_result(size_t r) { return r == ERR(E_dstSize_tooSmall) ? ERR(E_corruption_detected) : r; }

// The carried state at the start of a frame, before its first segment (what seg_tables sets up for `first`).
ZB_HD void seg_carry_init(SegCarry* c, u64 cap) {
    c->pos = 0; c->cap = cap; c->frameAt = 0; c->bad = 0; c->hasHuf = 0; c->hasFse = 0; c->hufLog = 0;
    c->rep[0] = 1; c->rep[1] = 4; c->rep[2] = 8;
    for (int t = 0; t < 3; t++) c->fseLog[t] = 0;
}

}  // namespace zb
