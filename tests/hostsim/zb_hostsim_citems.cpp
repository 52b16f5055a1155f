// zb_hostsim_citems.cpp -- TEST-ONLY host instantiation of zstdb200_compress_items_device's plan (zstd_jni_b200/csrc/zb_compress_items.cuh):
// the per-item count and bound, the scans, the capacity check, the parts of P slots with their boundaries and padding, the settling of each
// frame into its item, the packing and the results, as the k_citem_* kernels and k_scan_sizes compute them.  The frames themselves are
// stand-ins the caller gives per chunk.  tests/test_device_compress_items.py compiles it; it is never loaded by the product path.
#include <cstring>
#include <vector>
#include "../../zstd_jni_b200/csrc/zb_compress_items.cuh"

using namespace zb;

namespace {
// k_scan_sizes: exclusive scan of n sizes (errors count as 0) into n + 1 offsets
void scan_sizes(const u64* sizes, u64* offsets, size_t n) {
    u64 s = 0;
    for (size_t i = 0; i < n; i++) { offsets[i] = s; s += isErr((size_t)sizes[i]) ? 0 : sizes[i]; }
    offsets[n] = s;
}
}  // namespace

extern "C" {

// n items of sizes[i] bytes back to back from offset 0, cut into chunkSize pieces and compressed in parts of P slots into an output of
// `capacity` bytes (at address 0).  frame[j]: the frame result of chunk j (a size or an error code); padding slots get `padFrame`.
// Chunk j < jMax: its input [start[j], end[j]), its item, its frame's packed offset.  dstOff: n + 1, results: n.
// stats: {chunks, parts, padding slots, padding slots not empty at their part's end, padding frames packed}.
void zbc_plan(const unsigned long long* sizes, size_t n, unsigned long long chunkSize, unsigned long long capacity, unsigned P,
              const unsigned long long* frame, unsigned long long padFrame, unsigned long long* start, unsigned long long* end, unsigned* item,
              unsigned long long* packed, size_t jMax, unsigned long long* dstOff, unsigned long long* results, unsigned long long* stats) {
    std::vector<u64> srcOff(n + 1, 0), count(n), bound(n), first(n + 1), bounds(n + 1), errs(n);
    for (size_t i = 0; i < n; i++) srcOff[i + 1] = srcOff[i] + sizes[i];
    for (size_t i = 0; i < n; i++) {      // k_citem_count
        u64 const size = srcOff[i + 1] - srcOff[i];
        count[i] = chunk_count((size_t)size, (size_t)chunkSize); bound[i] = citem_bound(size, chunkSize); results[i] = 0; errs[i] = ~0ull;
    }
    scan_sizes(count.data(), first.data(), n);
    scan_sizes(bound.data(), bounds.data(), n);
    CItemCursor c{};      // k_citem_begin
    c.src = nullptr; c.srcOff = srcOff.data(); c.dst = nullptr; c.dstOff = (u64*)dstOff; c.results = (u64*)results; c.errs = errs.data();
    c.first = first.data(); c.chunkSize = chunkSize; c.n = (u32)n;
    citem_begin(c, first[n], bounds[n], capacity);
    std::vector<u64> slotOff(P + 1), sizesLead(P + 1), packedLead(P + 2, 0);
    std::vector<u32> slotItem(P);
    memset(stats, 0, 5 * sizeof(unsigned long long));
    stats[0] = c.m;
    auto next = [&]() {      // k_citem_next
        for (u32 k = 0; k < c.cnt; k++) {
            u32 const i = slotItem[k];
            if (c.at + k == c.first[i]) c.dstOff[i] = packedLead[1 + k];
        }
        bool const more = citem_advance(c, P, packedLead[P + 1]);
        sizesLead[0] = c.out;
        for (u32 k = 0; k <= P; k++) {
            u32 i = 0;
            slotOff[k] = citem_boundary(c, k, &i);
            if (k < c.cnt) slotItem[k] = i;
        }
        return more;
    };
    while (next()) {
        stats[1]++;
        for (u32 k = 0; k < P; k++) {      // the compress kernels' frames
            u64 const j = c.at + k;
            if (k < c.cnt) {
                if (j < jMax) { start[j] = slotOff[k]; end[j] = slotOff[k + 1]; item[j] = slotItem[k]; }
                sizesLead[1 + k] = frame[j];
            } else {
                stats[2]++;
                if (slotOff[k] != slotOff[c.cnt] || slotOff[k + 1] != slotOff[c.cnt]) stats[3]++;
                sizesLead[1 + k] = padFrame;
            }
        }
        for (u32 k = 0; k < P; k++) {      // k_citem_settle
            u64 const r = citem_slot_size(c, k, sizesLead[1 + k]);
            sizesLead[1 + k] = r;
            if (k >= c.cnt) continue;
            u32 const i = slotItem[k];
            u64 const key = citem_error_key(c.at + k, r);
            if (key != ~0ull) { if (key < c.errs[i]) c.errs[i] = key; } else c.results[i] += r;
        }
        scan_sizes(sizesLead.data(), packedLead.data(), P + 1);
        for (u32 k = 0; k < P; k++) {      // k_compact: the frames packed
            if (isErr((size_t)sizesLead[1 + k])) continue;
            if (k >= c.cnt) stats[4]++;
            else if (c.at + k < jMax) packed[c.at + k] = packedLead[1 + k];
        }
        for (u32 k = 0; k < c.cnt; k++) if (isErr((size_t)sizesLead[1 + k]) && c.at + k < jMax) packed[c.at + k] = packedLead[1 + k];
    }
    for (size_t i = 0; i <= n; i++) {      // k_citem_finish
        if (i == n || c.tooSmall) c.dstOff[i] = c.out;
        if (i < n) c.results[i] = citem_result(c, c.results[i], c.errs[i]);
    }
}

}
