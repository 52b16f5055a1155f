// zb_decode_list.cuh -- host side of the host-memory decompression calls: the decode list, which cuts items of several frames into their frames.
//
// An item item_walk lets split (zb_decode_fast.cuh) becomes one entry per frame -- a skippable frame too: it regenerates nothing, so
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
            bool ok = false;
            u32 const nf = item_walk(staged + srcOff[i], size, cap, nullptr, 0, &ok, magicless);
            if (!ok) continue;
            size_t const at = frames.size();
            frames.resize(at + nf);
            item_walk(staged + srcOff[i], size, cap, frames.data() + at, nf, &ok, magicless);
            u64 bytes = 0;      // what the item's frames regenerate: their declared sizes, or all of the capacity when the last declares none
            for (size_t k = at; k < at + nf; k++) if (!frames[k].skippable) bytes = frames[k].hasContentSize ? bytes + frames[k].contentSize : cap;
            if (bytes / nf < SPLIT_MIN_BYTES) { frames.resize(at); continue; }
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
                if (!f.skippable) d += f.hasContentSize ? f.contentSize : dstOff[i + 1] - d;
            }
        }
        L.src.push_back(srcOff[n]); L.dst.push_back(dstOff[n]); L.first[n] = m;
        L.m = m;
    } catch (const std::bad_alloc&) {
        whole();
    }
}

}  // namespace zb
