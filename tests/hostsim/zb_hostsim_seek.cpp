// zb_hostsim_seek.cpp -- TEST-ONLY host instantiation of the seek-table paths (zstd_jni_b200/csrc/zb_seek_table.cuh): the tables
// zstdb200_compress_items_device writes (zb_compress_items.cuh, as the k_citem_* kernels and k_citem_tables compute them, over stand-in
// frames), and zstdb200_decompress_ranges_device located through them (zb_decode_ranges.cuh: range_locate_any on one host lane or on
// the emulated 32-lane warp, range_fill_seek, the frames decoded by the fused decoder, range_entry_verify, the settling and the
// results).  tests/test_seek_table.py compiles it; it is never loaded by the product path.
#include <cstdlib>
#include <cstring>
#include <vector>
#include "../../zstd_jni_b200/csrc/zb_compress_items.cuh"
#include "../../zstd_jni_b200/csrc/zb_decode_ranges.cuh"
#include "simt_emu.h"

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

// The plan of one item of `size` bytes: out = {chunks, citem_seek_bound, citem_table_size, citem_count_key}.
void zbs_citem_item(unsigned long long size, unsigned long long chunkSize, unsigned E, unsigned long long* out) {
    u64 const k = chunk_count((size_t)size, (size_t)chunkSize);
    out[0] = k; out[1] = citem_seek_bound(size, chunkSize, E); out[2] = citem_table_size(k, E); out[3] = citem_count_key(k, E);
}

// n items of sizes[i] bytes, cut into chunkSize pieces, compressed in parts of P slots into `out` (capacity bytes) with tables of E-byte
// entries (0: none).  Chunk j's stand-in frame is frame[j] bytes (or an error code) of the byte j & 0xFF, its last four bytes xxh[j]
// when E is 12.  dstOff: n + 1, results: n.
void zbs_citems(const unsigned long long* sizes, size_t n, unsigned long long chunkSize, unsigned long long capacity, unsigned P, unsigned E,
                const unsigned long long* frame, const unsigned* xxh, unsigned char* out, unsigned long long* dstOff, unsigned long long* results) {
    std::vector<u64> srcOff(n + 1, 0), count(n), bound(n), first(n + 1), bounds(n + 1), errs(n);
    for (size_t i = 0; i < n; i++) srcOff[i + 1] = srcOff[i] + sizes[i];
    for (size_t i = 0; i < n; i++) {      // k_citem_count
        u64 const size = srcOff[i + 1] - srcOff[i];
        count[i] = chunk_count((size_t)size, (size_t)chunkSize); bound[i] = citem_seek_bound(size, chunkSize, E); results[i] = 0;
        errs[i] = citem_count_key(count[i], E);
    }
    scan_sizes(count.data(), first.data(), n);
    scan_sizes(bound.data(), bounds.data(), n);
    CItemCursor c{};      // k_citem_begin
    c.src = nullptr; c.srcOff = srcOff.data(); c.dst = out; c.dstOff = (u64*)dstOff; c.results = (u64*)results; c.errs = errs.data();
    c.first = first.data(); c.chunkSize = chunkSize; c.n = (u32)n; c.E = E;
    citem_begin(c, first[n], bounds[n], capacity);
    std::vector<u64> sizesLead(P + 1), rooms(P + 1), packed(P + 2, 0);
    std::vector<u32> slotItem(P), entries(E ? 2 * (size_t)citem_chunks_max(n, capacity, chunkSize, E) + 2 : 2);
    std::vector<u8> slot(compress_bound((size_t)chunkSize) + 64);
    auto next = [&]() {      // k_citem_next
        for (u32 k = 0; k < c.cnt; k++) {
            u32 const i = slotItem[k];
            if (c.at + k == c.first[i]) c.dstOff[i] = packed[1 + k];
        }
        bool const more = citem_advance(c, P, packed[P + 1]);
        rooms[0] = c.out;
        for (u32 k = 0; k < c.cnt; k++) { u32 i = 0; (void)citem_boundary(c, k, &i); slotItem[k] = i; }
        return more;
    };
    while (next()) {
        for (u32 k = 0; k < P; k++) {      // the compress kernels' frames, then k_citem_settle
            u64 const j = c.at + k;
            u64 const r = citem_slot_size(c, k, k < c.cnt ? frame[j] : 0);
            sizesLead[1 + k] = r;
            if (k >= c.cnt) { rooms[1 + k] = r; continue; }
            u32 const i = slotItem[k];
            u64 const key = citem_error_key(j, r);
            rooms[1 + k] = citem_slot_room(r, j + 1 == c.first[i + 1], citem_table_size(c.first[i + 1] - c.first[i], c.E));
            if (key != ~0ull) { if (key < c.errs[i]) c.errs[i] = key; continue; }
            c.results[i] += r;
            if (E) { entries[2 * j] = (u32)r; entries[2 * j + 1] = E == 12 ? xxh[j] : 0u; }
        }
        scan_sizes(rooms.data(), packed.data(), P + 1);
        for (u32 k = 0; k < c.cnt; k++) {      // k_compact
            u64 const j = c.at + k, r = sizesLead[1 + k];
            if (isErr((size_t)r)) continue;
            memset(slot.data(), (int)(j & 0xFF), (size_t)r);
            if (E == 12 && r >= 4) seek_store32(slot.data() + r - 4, xxh[j]);
            memcpy(out + packed[1 + k], slot.data(), (size_t)r);
        }
    }
    for (size_t i = 0; i <= n; i++) {      // k_citem_finish
        if (i == n || c.tooSmall) c.dstOff[i] = c.out;
        if (i < n) c.results[i] = citem_result(c, c.results[i] + citem_table_size(c.first[i + 1] - c.first[i], c.E), c.errs[i]);
    }
    if (E) {      // k_citem_tables
        for (u64 j = 0; j < c.m; j++) citem_table_entry(c, j, entries[2 * j], entries[2 * j + 1]);
        for (u32 i = 0; i < c.n && c.m; i++) citem_table_ends(c, i);
    }
}

// seek_table_read on item src[0, size): whether its table's structure is valid; t = {first entry's offset, k, E}.
int zbs_table_read(const void* src, size_t size, unsigned long long* t) {
    std::vector<u8> in(8, 0);
    in.insert(in.end(), (const u8*)src, (const u8*)src + size);
    in.resize(in.size() + 24, 0);
    SeekTable s{};
    bool const ok = seek_table_read(in.data() + 8, size, &s);
    t[0] = s.at; t[1] = s.k; t[2] = s.E;
    return ok ? 1 : 0;
}

// zbr_ranges (zb_hostsim_ranges.cpp) with seek tables: every request located by range_locate_any -- on one lane, or with emu on the
// emulated 32-lane warp -- then the parts; each entry's frame decoded by the fused decoder unless its check failed, verified against
// its table checksum, settled.  stats: [0] parts, [1] most entries in a part, [2] most partial entries in a part, [3] entries, [4] a
// scratch slot out of its part's S, [5] requests located through a table.
void zbs_ranges(const void* src, const unsigned long long* srcOff, size_t n, size_t m, const unsigned long long* items,
                const unsigned long long* begins, const unsigned long long* dstOff, unsigned P, unsigned S, int emu, void* dst,
                unsigned long long* results, unsigned long long* stats) {
    size_t const total = (size_t)(n ? srcOff[n] : 0);
    std::vector<u8> in(total + 64, 0);      // (slack on both sides, as the kernels' loads need)
    if (total) memcpy(in.data() + 16, src, total);
    const u8* const base = in.data() + 16;
    const u64* const so = (const u64*)srcOff; const u64* const dso = (const u64*)dstOff;
    std::vector<RangeReq> req(m);
    std::vector<u64> count(m), partial(m), first(m + 1, 0), pfirst(m + 1, 0);
    for (size_t r = 0; r < m; r++) {
        auto locate = [&](const auto& w) {
            range_locate_any(w, base, so, n, items[r], begins[r], dso[r + 1] - dso[r], &req[r], &count[r], &partial[r], (u64*)&results[r]);
        };
        if (emu) run_warp<32>([&](const WarpEmuT<32>& w) { locate(w); });
        else locate(WarpHost{});
    }
    for (size_t r = 0; r < m; r++) { first[r + 1] = first[r] + count[r]; pfirst[r + 1] = pfirst[r] + partial[r]; }
    std::vector<u8> out((size_t)dso[m] + 32);
    memcpy(out.data() + 16, dst, (size_t)dso[m]);
    u8* const o = out.data() + 16;
    std::vector<RangeSlot> slots(P);
    std::vector<u8> scratch((size_t)S * RANGE_PARTIAL_MAX + 64);
    DecShared* sh = (DecShared*)calloc(1, sizeof(DecShared));
    u8* dscratch = (u8*)calloc(1, BLOCKSIZE_MAX + 64);
    WarpHost w;
    for (int k = 0; k < 6; k++) stats[k] = 0;
    for (size_t r = 0; r < m; r++) stats[5] += (req[r].flags & RANGE_SEEK) != 0;
    RangePart p{};
    for (;;) {
        p = range_part(first.data(), pfirst.data(), req.data(), m, p.at + p.cnt, P, S);
        if (!p.cnt) break;
        for (u64 r = p.r0; r <= p.r1; r++) {
            if (first[r] == first[r + 1]) continue;
            u64 const i = items[r], b = begins[r];
            range_fill(base + so[i], (size_t)(so[i + 1] - so[i]), 0, b, range_end(b, dso[r + 1] - dso[r]), (u32)r, first[r], first[r + 1],
                       pfirst[r], &req[r], p, slots.data());
        }
        u64 parts = 0;
        for (u32 k = 0; k < p.cnt; k++) {
            RangeSlot const& s = slots[k];
            bool const part = s.scratch != NO_SCRATCH;
            if (part && s.scratch >= S) stats[4] = 1;
            parts += part;
            u8* const to = part ? scratch.data() + 16 + (size_t)(s.scratch % S) * RANGE_PARTIAL_MAX : o + dso[s.req] + s.to;
            u64 res = s.err ? 0 : decompress_item(w, *sh, base + so[items[s.req]] + s.pos, (size_t)s.size, to, (size_t)s.cs, dscratch, 0);
            res = range_entry_verify(w, s, res, to);
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
