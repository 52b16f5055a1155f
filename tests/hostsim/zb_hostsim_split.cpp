// zb_hostsim_split.cpp -- TEST-ONLY host instantiation of the device call's decode list (zstd_jni_b200/csrc/zb_decode_list.cuh): the
// per-item count, the scan, the fill and the part ranges the k_split_* kernels compute, the host plan they follow (plan_decode_list), the
// routing of the items left whole, and the settling of the entries' results.  tests/test_device_split.py compiles it; it is never
// loaded by the product path.
#include <cstdlib>
#include <cstring>
#include <vector>
#include "../../zstd_jni_b200/csrc/zb_decode_list.cuh"
#include "../../zstd_jni_b200/csrc/zb_decode_segment.cuh"

using namespace zb;

namespace {

// The items back to back with slack on both sides, as the kernels' loads need.
struct Staged {
    std::vector<u8> buf;
    explicit Staged(const void* src, size_t total) : buf(total + 64, 0) { memcpy(buf.data() + 16, src, total); }
    const u8* at(u64 off) const { return buf.data() + 16 + off; }
};

// k_split_count, k_scan_sizes and k_split_fill over n items, with a list of `max` entries: first[0 .. n] and the m entries listed.
struct DevicePlan {
    std::vector<u64> first, dst;
    std::vector<ItemFrame> frames;
    std::vector<u32> item;
    u64 m = 0;
    DevicePlan(const Staged& s, const u64* srcOff, const u64* dstOff, size_t n, u32 magicless, u64 max) : first(n + 1, 0) {
        for (size_t i = 0; i < n; i++)
            first[i + 1] = first[i] + split_device_count(s.at(srcOff[i]), (size_t)(srcOff[i + 1] - srcOff[i]), dstOff[i + 1] - dstOff[i], magicless);
        frames.resize(max); dst.resize(max); item.resize(max);
        for (size_t i = 0; i < n; i++) {
            if (!split_taken(first.data(), i, max)) continue;
            split_device_fill(s.at(srcOff[i]), (size_t)(srcOff[i + 1] - srcOff[i]), dstOff[i], dstOff[i + 1] - dstOff[i], magicless, (u32)i,
                              (u32)(first[i + 1] - first[i]), &frames[first[i]], &dst[first[i]], &item[first[i]]);
            m = first[i + 1] > m ? first[i + 1] : m;
        }
    }
    SplitRange range(u64 j, const u64* srcOff, const u64* dstOff) const { return split_range(frames.data(), dst.data(), item.data(), j, m, srcOff, dstOff); }
};

}  // namespace

extern "C" {

// The device plan of n items (list of `max` entries): taken[i] = item i is split; entry j < min(m, eMax): its input and output ranges and
// its item, e4[4 j ..] = {src, srcEnd, dst, dstEnd}.  Returns m.
unsigned long long zbs_device_plan(const void* src, const unsigned long long* srcOff, const unsigned long long* dstOff, size_t n, int magicless,
                                   unsigned long long max, unsigned char* taken, unsigned long long* e4, unsigned* eItem, size_t eMax) {
    Staged s(src, (size_t)srcOff[n]);
    DevicePlan P(s, (const u64*)srcOff, (const u64*)dstOff, n, (u32)magicless, max);
    for (size_t i = 0; i < n; i++) taken[i] = split_taken(P.first.data(), i, max) ? 1 : 0;
    for (u64 j = 0; j < P.m && j < eMax; j++) {
        SplitRange const r = P.range(j, (const u64*)srcOff, (const u64*)dstOff);
        e4[4 * j] = r.src; e4[4 * j + 1] = r.srcEnd; e4[4 * j + 2] = r.dst; e4[4 * j + 3] = r.dstEnd; eItem[j] = P.item[j];
    }
    return P.m;
}

// The host plan (plan_decode_list, the workspace always had): split[i], and entry j's ranges as above with its item, for j < min(m, eMax).
// Returns m (every item's entries, those kept whole included).
unsigned long long zbs_host_plan(const void* src, const unsigned long long* srcOff, const unsigned long long* dstOff, size_t n, int magicless,
                                 unsigned char* split, unsigned long long* e4, unsigned* eItem, size_t eMax) {
    Staged s(src, (size_t)srcOff[n]);
    DecodeList L;
    plan_decode_list(L, n, s.at(0), (const u64*)srcOff, (const u64*)dstOff, true, [](size_t) { return true; }, (u32)magicless);
    for (size_t i = 0; i < n; i++) {
        split[i] = L.split[i];
        for (size_t j = L.first[i]; j < L.first[i + 1] && j < eMax; j++) {
            e4[4 * j] = L.src[j]; e4[4 * j + 1] = L.src[j + 1]; e4[4 * j + 2] = L.dst[j]; e4[4 * j + 3] = L.dst[j + 1]; eItem[j] = (unsigned)i;
        }
    }
    return L.m;
}

// The routing of one item: its entries when the device splits it (split_device_count), else the blocks k_seg_route counts for the loop
// (seg_item_blocks, 0: not a loop candidate).
void zbs_route(const void* src, size_t size, unsigned long long cap, int magicless, unsigned* entries, unsigned long long* loopBlocks) {
    Staged s(src, size);
    *entries = split_device_count(s.at(0), size, cap, (u32)magicless);
    *loopBlocks = *entries ? 0 : seg_item_blocks(s.at(0), size, (u32)magicless);
}

// The device call on n items as far as the decode list goes: every entry of a split item decoded on its own (the fused decoder on the
// host, as the staged decoder regenerates the same bytes and codes), settled into its item (split_entry_stands), a marked item decoded
// again whole; every other item decoded whole.  status[i]: 0 kept whole, 1 split and settled, 2 split and decoded again.
void zbs_decode(const void* src, const unsigned long long* srcOff, const unsigned long long* dstOff, size_t n, int magicless, void* dst,
                unsigned long long* results, int* status) {
    Staged s(src, (size_t)srcOff[n]);
    u64 const max = (u64)1 << 20;
    DevicePlan P(s, (const u64*)srcOff, (const u64*)dstOff, n, (u32)magicless, max);
    std::vector<u8> out((size_t)dstOff[n] + 96, 0);      // (16 bytes of slack before the output)
    DecShared* S = (DecShared*)calloc(1, sizeof(DecShared));
    u8* scratch = (u8*)calloc(1, BLOCKSIZE_MAX + 64);
    WarpHost w;
    std::vector<u32> marks(n, 0);
    for (size_t i = 0; i < n; i++) { results[i] = 0; status[i] = split_taken(P.first.data(), i, max) ? 1 : 0; }
    for (u64 j = 0; j < P.m; j++) {
        SplitRange const r = P.range(j, (const u64*)srcOff, (const u64*)dstOff);
        u64 const res = decompress_item(w, *S, s.at(r.src), (size_t)(r.srcEnd - r.src), out.data() + 16 + r.dst, (size_t)(r.dstEnd - r.dst), scratch,
                                        (u32)magicless);
        u32 const i = P.item[j];
        if (split_entry_stands(P.frames[j], res)) results[i] += res; else marks[i] = 1;
    }
    for (size_t i = 0; i < n; i++) {
        if (status[i] == 1 && !marks[i]) continue;
        if (status[i] == 1) status[i] = 2;
        results[i] = decompress_item(w, *S, s.at(srcOff[i]), (size_t)(srcOff[i + 1] - srcOff[i]), out.data() + 16 + dstOff[i],
                                     (size_t)(dstOff[i + 1] - dstOff[i]), scratch, (u32)magicless);
    }
    memcpy(dst, out.data() + 16, (size_t)dstOff[n]);
    free(S); free(scratch);
}

}
