// zb_hostsim_ranges.cpp -- TEST-ONLY host instantiation of zstdb200_decompress_ranges_device (zstd_jni_b200/csrc/zb_decode_ranges.cuh):
// every request located (range_locate), the scans of its entries and partial entries, the parts of at most P entries and S partial ones
// (range_part), the slots every request writes (range_fill), each slot decoded on its own by the fused decoder (the staged decoder gives
// the same bytes and codes), settled (range_entry_key), a partial slot's slice copied out, and the results (range_result).
// tests/test_device_ranges.py compiles it; it is never loaded by the product path.
#include <cstdlib>
#include <cstring>
#include <vector>
#include "../../zstd_jni_b200/csrc/zb_decode_ranges.cuh"

using namespace zb;

extern "C" {

// The call on n items (src, srcOff: n + 1) and m requests (items, begins, dstOff: m + 1) in parts of P entries, at most S of them
// partial.  dst (dstOff[m] bytes) is written where the call writes; results[m].  stats: [0] parts, [1] most entries in a part, [2] most
// partial entries in a part, [3] entries, [4] a scratch slot out of its part's S (0: never).
void zbr_ranges(const void* src, const unsigned long long* srcOff, size_t n, size_t m, const unsigned long long* items,
                const unsigned long long* begins, const unsigned long long* dstOff, unsigned P, unsigned S, int magicless, void* dst,
                unsigned long long* results, unsigned long long* stats) {
    size_t const total = (size_t)(n ? srcOff[n] : 0);
    std::vector<u8> in(total + 64, 0);      // (slack on both sides, as the kernels' loads need)
    if (total) memcpy(in.data() + 16, src, total);
    const u8* const base = in.data() + 16;
    const u64* const so = (const u64*)srcOff; const u64* const dso = (const u64*)dstOff;
    std::vector<RangeReq> req(m);
    std::vector<u64> count(m), partial(m), first(m + 1, 0), pfirst(m + 1, 0);
    for (size_t r = 0; r < m; r++)
        range_locate(base, so, n, items[r], begins[r], dso[r + 1] - dso[r], (u32)magicless, &req[r], &count[r], &partial[r], (u64*)&results[r]);
    for (size_t r = 0; r < m; r++) { first[r + 1] = first[r] + count[r]; pfirst[r + 1] = pfirst[r] + partial[r]; }
    std::vector<u8> out((size_t)dso[m] + 32);
    memcpy(out.data() + 16, dst, (size_t)dso[m]);
    u8* const o = out.data() + 16;
    std::vector<RangeSlot> slots(P);
    std::vector<u8> scratch((size_t)S * RANGE_PARTIAL_MAX + 64);
    DecShared* sh = (DecShared*)calloc(1, sizeof(DecShared));
    u8* dscratch = (u8*)calloc(1, BLOCKSIZE_MAX + 64);
    WarpHost w;
    for (int k = 0; k < 5; k++) stats[k] = 0;
    RangePart p{};
    for (;;) {
        p = range_part(first.data(), pfirst.data(), req.data(), m, p.at + p.cnt, P, S);
        if (!p.cnt) break;
        for (u64 r = p.r0; r <= p.r1; r++) {
            if (first[r] == first[r + 1]) continue;
            u64 const i = items[r], b = begins[r];
            range_fill(base + so[i], (size_t)(so[i + 1] - so[i]), (u32)magicless, b, range_end(b, dso[r + 1] - dso[r]), (u32)r, first[r], first[r + 1],
                       pfirst[r], &req[r], p, slots.data());
        }
        u64 parts = 0;
        for (u32 k = 0; k < p.cnt; k++) {
            RangeSlot const& s = slots[k];
            bool const part = s.scratch != NO_SCRATCH;
            if (part && s.scratch >= S) stats[4] = 1;
            parts += part;
            u8* const to = part ? scratch.data() + 16 + (size_t)(s.scratch % S) * RANGE_PARTIAL_MAX : o + dso[s.req] + s.to;
            u64 const res = decompress_item(w, *sh, base + so[items[s.req]] + s.pos, (size_t)s.size, to, (size_t)s.cs, dscratch, (u32)magicless);
            u64 const key = range_entry_key(s, res);
            if (key != ~0ull) { if (key < req[s.req].err) req[s.req].err = key; }
            else if (part) memmove(o + dso[s.req] + s.to, to + s.from, s.len);
        }
        stats[0]++; stats[3] += p.cnt;
        if (p.cnt > stats[1]) stats[1] = p.cnt;
        if (parts > stats[2]) stats[2] = parts;
    }
    for (size_t r = 0; r < m; r++) results[r] = range_result(req[r].err, results[r]);
    memcpy(dst, o, (size_t)dso[m]);
    free(sh); free(dscratch);
}

}
