// zb_hostsim_seg.cpp -- TEST-ONLY host instantiation of the segment decoder (zstd_jni_b200/csrc/zb_decode_segment.cuh): the stages the
// k_seg_* kernels run, driven from the host with the block order shuffled, segment cuts anywhere and the carried state passed between
// them.  Never loaded by the product path.
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include <vector>
#include "../../zstd_jni_b200/csrc/zb_decode_segment.cuh"
#include "simt_emu.h"

using namespace zb;

extern "C" {

// One item through the segment stages: segments of segBlocks blocks (0: the whole frame in one), the per-block stages and the byte
// links in an order shuffled by `seed`, stages A and D on the 32-lane emulator when emu != 0.  *status: 0 decoded (the size is
// returned), 1 deferred to the fused decoder, 2 not a frame the segment decoder takes.
size_t zbs_decompress(void* dst, size_t cap, const void* src, size_t size, unsigned segBlocks, unsigned seed, int emu, int* status) {
    std::vector<u8> in(size + 64), out(cap + 64);
    memcpy(in.data() + 16, src, size);
    const u8* const frame = in.data() + 16;
    u8* const o = out.data() + 16;
    FrameHeader fh; u32 xxh = 0;
    u32 const n = seg_walk(frame, size, &fh, nullptr, &xxh);
    if (!n) { *status = 2; return 0; }
    std::vector<u64> refs(n);
    seg_walk(frame, size, &fh, refs.data(), &xxh);
    u32 const B = segBlocks && segBlocks < n ? segBlocks : n;
    constexpr size_t LS = BLOCKSIZE_MAX + 64;
    std::vector<SegBlock> blocks(B);
    std::vector<u16> huf((size_t)B * SEG_HUF_ENTRIES);
    std::vector<u32> fse((size_t)B * FAST_FSE_ENTRIES), offs((size_t)B * FAST_MAXS), link((size_t)B * BLOCKSIZE_MAX);
    std::vector<u8> lit((size_t)B * LS);
    std::vector<u64> seqs((size_t)B * FAST_MAXS);
    SegCarry* c = (SegCarry*)calloc(1, sizeof(SegCarry));
    DecShared* S = (DecShared*)calloc(1, sizeof(DecShared));
    std::mt19937 rng(seed);
    WarpHost h;
    for (u32 first = 0; first < n && !c->bad; first += B) {
        u32 const cnt = n - first < B ? n - first : B;
        std::vector<u32> order(cnt);
        for (u32 j = 0; j < cnt; j++) order[j] = j;
        std::shuffle(order.begin(), order.end(), rng);
        for (u32 j : order) {
            u32 const off = (u32)refs[first + j], bh = (u32)(refs[first + j] >> 32);
            auto prep = [&](const auto& w) { seg_prepare(w, *S, frame, off, bh, fh.blockSizeMax, &blocks[j], &huf[(size_t)j * SEG_HUF_ENTRIES], &fse[(size_t)j * FAST_FSE_ENTRIES]); };
            if (emu) run_warp<32>([&](const WarpEmuT<32>& w) { prep(w); }); else prep(h);
        }
        seg_tables(blocks.data(), cnt, c, first == 0, cap);
        if (c->bad) break;
        for (u32 j : order) for (int k = 0; k < 4; k++) seg_huf(blocks.data(), j, k, frame, huf.data(), c, &lit[(size_t)j * LS]);
        for (u32 j : order) seg_seq(blocks.data(), j, frame, fse.data(), c, &seqs[(size_t)j * FAST_MAXS], &offs[(size_t)j * FAST_MAXS]);
        seg_scan(blocks.data(), cnt, c, fh.blockSizeMax);
        if (c->bad) break;
        for (u32 j : order) seg_offsets(blocks.data(), j, &seqs[(size_t)j * FAST_MAXS], &offs[(size_t)j * FAST_MAXS]);
        seg_carry_tables(h, blocks.data(), huf.data(), fse.data(), c);
        u64 const segStart = blocks[0].out;
        for (u32 j : order) {
            auto fill = [&](const auto& w, SegRec* R) { seg_fill(w, R, blocks.data(), j, frame, &lit[(size_t)j * LS], &seqs[(size_t)j * FAST_MAXS], &offs[(size_t)j * FAST_MAXS], o, segStart, link.data(), c); };
            SegRec R[32];
            if (emu) run_warp<32>([&](const WarpEmuT<32>& w) { fill(w, R); }); else fill(h, R);
        }
        if (c->bad) break;
        std::vector<u32> bytes((size_t)(c->pos - segStart));
        for (size_t p = 0; p < bytes.size(); p++) bytes[p] = (u32)p;
        std::shuffle(bytes.begin(), bytes.end(), rng);
        for (u32 p : bytes) o[segStart + p] = seg_jump(link.data(), p);
    }
    bool ok = !c->bad && (!fh.hasContentSize || c->pos == fh.contentSize) && (!fh.checksum || (u32)xxh64(o, (size_t)c->pos) == xxh);
    size_t const r = ok ? (size_t)c->pos : 0;
    if (ok) memcpy(dst, o, r);
    *status = ok ? 0 : 1;
    free(c); free(S);
    return r;
}

// The repcode summaries against the serial walk: `n` random blocks of up to `maxSeq` selectors each (idx 0..4; new offsets small enough
// to run the history through zero and past it), from a random start history that may hold 0xFFFFFFFF -- a corrupted one.  The summary
// of every block, applied in block order, must give the history the serial walk has at every block start.  Returns the mismatches.
unsigned zbs_rep_check(unsigned seed, unsigned n, unsigned maxSeq) {
    std::mt19937 rng(seed);
    unsigned bad = 0;
    auto pick = [&](u32 lo, u32 hi) { return std::uniform_int_distribution<u32>(lo, hi)(rng); };
    u32 serial[3], scanned[3];
    for (int s = 0; s < 3; s++) { u32 const v = pick(0, 3) == 0 ? 0xFFFFFFFFu - pick(0, 2) : pick(1, 5); serial[s] = scanned[s] = v; }
    for (unsigned b = 0; b < n; b++) {
        u32 const m = pick(0, maxSeq);
        RepSym sum[3] = { { 0, 0 }, { 1, 0 }, { 2, 0 } };
        for (u32 k = 0; k < m; k++) {
            // a sequence's offset code (0, 1 or more extra bits), whether its litLength is 0, the extra bit, the new offset
            u32 const ofBits = pick(0, 2), ll0 = pick(0, 1), ofVal = ofBits == 1 ? pick(0, 1) : 0, v = pick(1, 4);
            // the fused decoder's serial walk (decode_block, zb_decode.cuh)
            if (ofBits > 1) { serial[2] = serial[1]; serial[1] = serial[0]; serial[0] = v; }
            else if (ofBits == 0) { u32 const offset = ll0 ? serial[1] : serial[0]; serial[1] = ll0 ? serial[0] : serial[1]; serial[0] = offset; }
            else {
                u32 const i = 1 + ll0 + ofVal;
                u32 temp = i == 3 ? serial[0] - 1 : (i == 1 ? serial[1] : serial[2]);
                temp -= !temp;
                if (i != 1) serial[2] = serial[1];
                serial[1] = serial[0]; serial[0] = temp;
            }
            // the selector seg_seq keeps (SeqValue::take_if)
            rep_step_sym(sum, ofBits > 1 ? 4u : ofBits + ll0 + ofVal, v);
        }
        u32 nr[3];
        for (int s = 0; s < 3; s++) nr[s] = rep_eval(sum[s], scanned);
        for (int s = 0; s < 3; s++) scanned[s] = nr[s];
        for (int s = 0; s < 3; s++) if (scanned[s] != serial[s]) bad++;
    }
    return bad;
}

}
