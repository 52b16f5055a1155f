// zb_hostsim_loop.cpp -- TEST-ONLY host instantiation of the segment loop of zstdb200_decompress_device (zstd_jni_b200/csrc/
// zb_decode_segment.cuh): the items routed by seg_item_blocks, their blocks walked into segments of B blocks that cross frame and item
// boundaries (seg_walk_segment), and every stage of a segment in the order the loop's graph runs them, the per-block stages over the
// blocks in an order shuffled by `seed`.  Never loaded by the product path.
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <random>
#include <vector>
#include "../../zstd_jni_b200/csrc/zb_decode_segment.cuh"
#include "simt_emu.h"

using namespace zb;

extern "C" {

// The blocks of an item the loop takes (0: the item stays with the other decoders).
unsigned long long zbl_item_blocks(const void* src, size_t size, int magicless) { return seg_item_blocks((const u8*)src, size, (u32)magicless); }

// The least blocks of an item on the loop when the n candidates have blocks[0 .. n) blocks and the fused kernel `warps` warps.
unsigned long long zbl_min_blocks(const unsigned long long* blocks, size_t n, unsigned long long warps) {
    u32 cnt[SEG_BUCKETS] = {}, mx[SEG_BUCKETS] = {};
    u64 sum[SEG_BUCKETS] = {};
    for (size_t i = 0; i < n; i++) {
        u32 const k = seg_bucket(blocks[i]);
        cnt[k]++; sum[k] += blocks[i]; if (blocks[i] > mx[k]) mx[k] = (u32)blocks[i];
    }
    return seg_loop_min_blocks(cnt, sum, mx, warps);
}

// n items (item i at src[srcOff[i], srcOff[i+1]), its output at dst[dstOff[i], dstOff[i+1])) through the loop with segments of B
// blocks, stages A and D and the frame ends on the 32-lane emulator when emu != 0.  status[i]: 0 the loop decoded it (results[i] = its
// size), 1 the loop marked it for the fused decoder, 2 not routed to the loop.  Returns the number of segments.
unsigned zbl_loop(const void* src, const unsigned long long* srcOff, size_t n, void* dst, const unsigned long long* dstOff,
                  unsigned long long* results, int* status, unsigned B, int magicless, unsigned seed, int emu) {
    std::vector<u32> list, bad(n, 0);
    for (size_t i = 0; i < n; i++) {
        bool const loop = seg_item_blocks((const u8*)src + srcOff[i], (size_t)(srcOff[i + 1] - srcOff[i]), (u32)magicless) != 0;
        status[i] = loop ? 0 : 2;
        results[i] = 0;
        if (loop) list.push_back((u32)i);
    }
    std::mt19937 rng(seed);
    std::shuffle(list.begin(), list.end(), rng);      // the device list is in the order the routing threads append
    SegCursor cur{};
    cur.src = (const u8*)src; cur.srcOff = (const u64*)srcOff; cur.dst = (u8*)dst; cur.dstOff = (const u64*)dstOff; cur.results = (u64*)results;
    cur.itemBad = bad.data(); cur.list = list.data(); cur.count = (u32)list.size(); cur.magicless = (u32)magicless; cur.first = 1;
    constexpr size_t LS = BLOCKSIZE_MAX + 64;
    std::vector<u64> refs(B);
    std::vector<SegLoc> loc(B);
    std::vector<SegBlock> blocks(B);
    std::vector<u16> huf((size_t)B * SEG_HUF_ENTRIES);
    std::vector<u32> fse((size_t)B * FAST_FSE_ENTRIES), offs((size_t)B * FAST_MAXS), link((size_t)B * BLOCKSIZE_MAX);
    std::vector<u8> lit((size_t)B * LS);
    std::vector<u64> seqs((size_t)B * FAST_MAXS);
    SegCarry* c = (SegCarry*)calloc(1, sizeof(SegCarry));
    DecShared* S = (DecShared*)calloc(1, sizeof(DecShared));
    WarpHost h;
    auto in = [&](u32 j) { return (const u8*)src + srcOff[loc[j].item]; };
    auto out = [&](u32 j) { return (u8*)dst + dstOff[loc[j].item]; };
    unsigned segments = 0;
    for (u32 cnt; (cnt = seg_walk_segment(&cur, B, refs.data(), loc.data())) != 0; segments++) {
        std::vector<u32> order(cnt);
        for (u32 j = 0; j < cnt; j++) order[j] = j;
        std::shuffle(order.begin(), order.end(), rng);
        for (u32 j : order) {
            auto prep = [&](const auto& w) { seg_prepare(w, *S, in(j), (u32)refs[j], (u32)(refs[j] >> 32), loc[j].blockSizeMax, &blocks[j],
                                                         &huf[(size_t)j * SEG_HUF_ENTRIES], &fse[(size_t)j * FAST_FSE_ENTRIES]); };
            if (emu) run_warp<32>([&](const WarpEmuT<32>& w) { prep(w); }); else prep(h);
        }
        seg_tables(blocks.data(), cnt, c, false, 0, loc.data(), bad.data());
        for (u32 j : order) {
            if (bad[loc[j].item]) continue;
            for (int k = 0; k < 4; k++) seg_huf(blocks.data(), j, k, in(j), huf.data(), c, &lit[(size_t)j * LS]);
            seg_seq(blocks.data(), j, in(j), fse.data(), c, &seqs[(size_t)j * FAST_MAXS], &offs[(size_t)j * FAST_MAXS]);
        }
        seg_scan(blocks.data(), cnt, c, 0, loc.data(), bad.data());
        for (u32 j : order) if (!bad[loc[j].item]) seg_offsets(blocks.data(), j, &seqs[(size_t)j * FAST_MAXS], &offs[(size_t)j * FAST_MAXS]);
        seg_carry_tables(h, blocks.data(), huf.data(), fse.data(), c);
        for (u32 j : order) {
            if (bad[loc[j].item]) continue;
            auto fill = [&](const auto& w, SegRec* R) { seg_fill(w, R, blocks.data(), j, in(j), &lit[(size_t)j * LS], &seqs[(size_t)j * FAST_MAXS],
                                                                 &offs[(size_t)j * FAST_MAXS], out(j), ~0ull, ~0ull, link.data(), &bad[loc[j].item]); };
            SegRec R[32];
            if (emu) run_warp<32>([&](const WarpEmuT<32>& w) { fill(w, R); }); else fill(h, R);
        }
        // the link map entries in shuffled order, each written to its block's item (k_seg_jump)
        std::vector<u32> entries(c->links);
        for (u32 p = 0; p < c->links; p++) entries[p] = p;
        std::shuffle(entries.begin(), entries.end(), rng);
        for (u32 p : entries) {
            u32 j = 0;
            while (j + 1 < cnt && blocks[j + 1].linkAt + (blocks[j + 1].out - blocks[j + 1].segAt) <= p) j++;
            if (!bad[loc[j].item]) out(j)[blocks[j].segAt + (p - blocks[j].linkAt)] = seg_jump(link.data(), p);
        }
        for (u32 j : order) {
            if (!(loc[j].flags & LOC_END) || bad[loc[j].item]) continue;
            u64 end = 0;
            auto fin = [&](const auto& w) { end = seg_frame_end(w, blocks.data(), j, loc[j], out(j), &bad[loc[j].item]); };
            if (emu) run_warp<32>([&](const WarpEmuT<32>& w) { fin(w); }); else fin(h);
            results[loc[j].item] = std::max<unsigned long long>(results[loc[j].item], end);
        }
    }
    for (size_t i = 0; i < n; i++) if (status[i] == 0 && bad[i]) status[i] = 1;
    free(c); free(S);
    return segments;
}

}
