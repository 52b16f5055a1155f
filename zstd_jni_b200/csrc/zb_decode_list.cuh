// zb_decode_list.cuh -- the decode list, which cuts items of several frames into their frames: planned on the host for the host-memory
// decompression calls (plan_decode_list), on the GPU for the device-memory call (split_device_*, kernels k_split_* in zb_capi.cu).
//
// An item the split rule takes (split_entries) becomes one entry per frame -- a skippable frame too: it regenerates nothing, so
// its capacity is 0 -- output at the item's output plus the declared sizes of the frames before it, capacity its own declared size (the
// last entry: the rest of the item's).  Every other item is one entry.  The staged, segment and fused decoders then run over the entries
// as over items, so every entry costs the staged decoder's per-item workspace (about 0.5 MB, per launch part of at most
// LAUNCH_MAX_FRAMES entries).  Hence two limits, after which the items stay whole, as with dec_pipeline 0:
//   - an item is split only when it regenerates at least SPLIT_MIN_BYTES per entry on average (a stream of many tiny or empty frames
//     would cost far more workspace than it has bytes);
//   - the call's `reserve(m)` must get the workspaces of m entries; when it cannot (or the host lists cannot be had), no item is split.
#pragma once
#include <new>
#include <vector>

#include "zb_decode_fast.cuh"

namespace zb {

constexpr u64 SPLIT_MIN_BYTES = 32768;      // bytes regenerated per entry, on average, by an item that is split (the staged workspace
                                            // of an entry is about 15 times that)

// The split rule: the number of entries item src[0, size) of output capacity `cap` is cut into -- its frames -- or 0 when it is decoded
// whole.  An item is split when item_walk lets it be and it regenerates at least SPLIT_MIN_BYTES per entry on average.
// *mostBlocks: the most blocks of one of its frames.
ZB_HDN u32 split_entries(const u8* src, size_t size, u64 cap, u32 magicless, u32* mostBlocks = nullptr) {
    bool ok = false; u64 bytes = 0; u32 most = 0;
    u32 const nf = item_walk(src, size, cap, nullptr, 0, &ok, magicless, &bytes, &most);
    if (mostBlocks) *mostBlocks = most;
    return ok && bytes / nf >= SPLIT_MIN_BYTES ? nf : 0;
}

// ---------------------------------------------------------------------------------------- the device call's list
// zstdb200_decompress_device plans on the GPU: every item is counted (split_device_count), the counts are scanned into each item's first
// entry, and the frames of every item taken are written to its entries (split_device_fill) -- plan_decode_list's entries in its order,
// less those of the items kept whole.  The list holds at most `max` entries; an item whose entries would end beyond it is not taken.
// The staged pipeline decodes the entries in parts (split_range), and each entry's result settles into its item (split_entry_stands):
// the item's result is the sum of its entries', or the item is marked and the fused decoder decodes it again whole.

// The entries of an item the device call splits: the split rule's, when every zstd frame of the item is one block (skippable frames
// allowed; frames of several blocks stay with the segment loop).  0: the item is routed as without splitting.
ZB_HDN u32 split_device_count(const u8* src, size_t size, u64 cap, u32 magicless) {
    u32 most = 0;
    u32 const nf = split_entries(src, size, cap, magicless, &most);
    return most == 1 ? nf : 0;
}

// Whether item i is split: it has entries [first[i], first[i + 1]) and they fit the list of `max` entries (first null: none is).
ZB_HD bool split_taken(const u64* first, u64 i, u64 max) { return first && first[i + 1] > first[i] && first[i + 1] <= max; }

// The output offset of the entry after frame f's, which starts at d in an item whose output ends at `end`: a skippable frame takes
// nothing, a frame its declared size, a frame without one the rest of the item's capacity.
ZB_HD u64 split_next_dst(const ItemFrame& f, u64 d, u64 end) { return f.skippable ? d : f.hasContentSize ? d + f.contentSize : end; }

// The `count` entries of item i (input src[0, size), output at dstAt of capacity cap): its frames to frames[0 .. count), the output
// offset of each to dst[0 .. count), i to item[0 .. count).
ZB_HDN void split_device_fill(const u8* src, size_t size, u64 dstAt, u64 cap, u32 magicless, u32 i, u32 count, ItemFrame* frames, u64* dst,
                              u32* item) {
    bool ok = false;
    item_walk(src, size, cap, frames, count, &ok, magicless);
    u64 d = dstAt;
    for (u32 q = 0; q < count; q++) {
        dst[q] = d; item[q] = i;
        d = split_next_dst(frames[q], d, dstAt + cap);
    }
}

// Entry j of the m listed: its input [src, srcEnd) and output [dst, dstEnd), offsets in the call's buffers (srcOff, dstOff: the items').
// An item's last entry ends where the item does.
struct SplitRange { u64 src, srcEnd, dst, dstEnd; };
ZB_HD SplitRange split_range(const ItemFrame* frames, const u64* dst, const u32* item, u64 j, u64 m, const u64* srcOff, const u64* dstOff) {
    u32 const i = item[j];
    SplitRange r;
    r.src = srcOff[i] + frames[j].srcOff; r.srcEnd = r.src + frames[j].srcSize;
    r.dst = dst[j]; r.dstEnd = j + 1 < m && item[j + 1] == i ? dst[j + 1] : dstOff[i + 1];
    return r;
}

// Whether an entry's result r stands for its frame: no error, and exactly the declared size (a skippable frame: nothing; a last frame
// without a declared size: whatever fit).  When one does not, its item is decoded again whole.
ZB_HD bool split_entry_stands(const ItemFrame& f, u64 r) {
    return !isErr((size_t)r) && (f.skippable ? r == 0 : !f.hasContentSize || r == f.contentSize);
}

struct DecodeList {
    size_t m = 0;                        // entries
    std::vector<u8> split;               // per item: cut into its frames
    std::vector<u64> src, dst;           // entry j: input [src[j], src[j + 1]), output [dst[j], dst[j + 1]) (m + 1 each)
    std::vector<size_t> first;           // item i: entries [first[i], first[i + 1])
    std::vector<ItemFrame> frame;        // the frame of each entry of a split item (unused for the others)
    std::vector<ItemFrame> walked;       // planning scratch: the frames of the items to split, in item order
    std::vector<u32> count;              // ... and how many each has
};

// n items back to back at `staged`: item i's input [srcOff[i], srcOff[i + 1]), its output [dstOff[i], dstOff[i + 1]) (both n + 1 long).
// pipeline false: every item whole.  reserve(m) -> whether the workspaces of m entries could be had.  magicless: the items are in the
// ZSTD_f_zstd1_magicless format.  The list's vectors keep their storage from one plan to the next.
template <class Reserve>
void plan_decode_list(DecodeList& L, size_t n, const u8* staged, const u64* srcOff, const u64* dstOff, bool pipeline, Reserve reserve,
                      u32 magicless = 0) {
    auto whole = [&] {
        L.m = n; L.split.assign(n, 0); L.frame.clear();
        L.src.assign(srcOff, srcOff + n + 1); L.dst.assign(dstOff, dstOff + n + 1);
        L.first.resize(n + 1); for (size_t i = 0; i <= n; i++) L.first[i] = i;
    };
    whole();
    if (!pipeline) return;
    try {
        std::vector<ItemFrame>& frames = L.walked;
        std::vector<u32>& count = L.count;
        frames.clear(); count.assign(n, 0);
        size_t m = n;
        for (size_t i = 0; i < n; i++) {
            size_t const size = (size_t)(srcOff[i + 1] - srcOff[i]);
            u64 const cap = dstOff[i + 1] - dstOff[i];
            u32 const nf = split_entries(staged + srcOff[i], size, cap, magicless);
            if (!nf) continue;
            size_t const at = frames.size();
            frames.resize(at + nf);
            bool ok = false;
            item_walk(staged + srcOff[i], size, cap, frames.data() + at, nf, &ok, magicless);
            L.split[i] = 1; count[i] = nf; m += nf - 1;
        }
        if (m == n) return;
        if (m > 0x7FFFFFFFull || !reserve(m)) { whole(); return; }
        L.src.clear(); L.dst.clear(); L.frame.resize(m);
        size_t k = 0;
        for (size_t i = 0; i < n; i++) {
            L.first[i] = L.src.size();
            if (!L.split[i]) { L.src.push_back(srcOff[i]); L.dst.push_back(dstOff[i]); continue; }
            u64 d = dstOff[i];
            for (u32 q = 0; q < count[i]; q++) {
                ItemFrame const& f = frames[k++];
                L.frame[L.src.size()] = f;
                L.src.push_back(srcOff[i] + f.srcOff); L.dst.push_back(d);
                d = split_next_dst(f, d, dstOff[i + 1]);
            }
        }
        L.src.push_back(srcOff[n]); L.dst.push_back(dstOff[n]); L.first[n] = m;
        L.m = m;
    } catch (const std::bad_alloc&) {
        whole();
    }
}

}  // namespace zb
