// zb_compress_items.cuh -- the plan of zstdb200_compress_items_device: items in device memory cut into chunkSize pieces on the GPU, each
// piece one frame (the stream ZSTD_compress2 writes with ZSTDB200_c_multiFrame), compressed in parts of P chunks and packed in item order.
// The kernels k_citem_* in zb_capi.cu are thin wrappers of these functions; tests/hostsim/zb_hostsim_citems.cpp runs them on the host.
//
// Every item is counted -- its chunks (chunk_count) and their summed compress bound (citem_bound) -- the counts are scanned into each
// item's first chunk and the bounds into their total, which the capacity must reach (citem_begin).  A part is P slots (citem_advance): the
// next chunks, and past the last of them zero-length chunks at the end offset (citem_boundary), so the slot boundaries are monotone.  Once
// the part's frames are written, the padding frames are dropped (citem_slot_size), each chunk's frame adds its size to its item or records
// its error (citem_error_key), the frames kept are packed after the bytes of the parts before, and the next part is planned.
//
// With seek tables (E, the entry size, nonzero) every item is followed by its table (zb_seek_table.cuh).  An item's bound grows by its
// table (citem_seek_bound), and an item of more chunks than a table may list fails (citem_count_key).  Each chunk's frame keeps its size
// and checksum in the workspace; the last chunk of an item packs as its frame plus the item's table (citem_slot_room), so the packing
// leaves room for every table of an item whose last chunk is in the part.  Once every part has run, the tables are written in parallel:
// entry by entry (citem_table_entry) and, per item, header and footer (citem_table_ends), before the next item's first frame.
#pragma once
#include "zb_encode.cuh"
#include "zb_seek_table.cuh"

namespace zb {

// Chunks of an item of srcSize bytes: an empty item is one empty frame.
ZB_HD size_t chunk_count(size_t srcSize, size_t chunkSize) { return srcSize ? (srcSize + chunkSize - 1) / chunkSize : 1; }

// The summed ZSTD_compressBound of an item's chunks: the room its frames may need.
ZB_HD u64 citem_bound(u64 size, u64 chunkSize) {
    u64 const rest = size % chunkSize;
    return size / chunkSize * compress_bound((size_t)chunkSize) + (rest || !size ? compress_bound((size_t)rest) : 0);
}

// The call and the part being compressed.
struct CItemCursor {
    const u8* src; const u64* srcOff; u8* dst; u64* dstOff; u64* results;      // the call's arguments
    u64* errs;                   // per item the least citem_error_key of its frames (~0: none)
    const u64* first;            // item i's chunks: [first[i], first[i + 1])
    u64 chunkSize; u32 n;
    u32 tooSmall;                // the capacity is short of the bound: no part runs
    u64 m;                       // chunks to compress (0 when tooSmall)
    u64 at; u32 cnt;             // the part: chunks [at, at + cnt)
    u64 out;                     // bytes packed by the parts before it
    u32 E;                       // seek-table entry size (8 or 12), 0: no tables
};

// The bytes of the table after an item of k chunks: none without tables, or when the item has more chunks than a table may list.
ZB_HD u64 citem_table_size(u64 k, u32 E) { return E && k <= SEEK_FRAMES_MAX ? seek_table_size(k, E) : 0; }

// The room an item of `size` bytes may need: its chunks' bound, and its table.
ZB_HD u64 citem_seek_bound(u64 size, u64 chunkSize, u32 E) {
    return citem_bound(size, chunkSize) + (E ? seek_table_size(chunk_count((size_t)size, (size_t)chunkSize), E) : 0);
}

// The error key an item of k chunks starts with: frameIndex_tooLarge, ahead of every frame's, when it needs a table of more entries
// than one may hold; else none (~0).
ZB_HD u64 citem_count_key(u64 k, u32 E) { return E && k > SEEK_FRAMES_MAX ? (u64)E_frameIndex_tooLarge : ~0ull; }

// Chunks a call may hold when its capacity reaches the bound, for the per-chunk workspace of its tables: a full chunk's bound exceeds
// chunkSize, and every chunk's bound and entry take at least 64 + E bytes.
ZB_HD u64 citem_chunks_max(u64 n, u64 capacity, u64 chunkSize, u32 E) {
    u64 const a = n + capacity / chunkSize, b = capacity / (64 + E);
    return a < b ? a : b;
}

// The cursor before the first part, for m chunks whose bounds sum to `bound`.
ZB_HD void citem_begin(CItemCursor& c, u64 m, u64 bound, u64 capacity) {
    c.tooSmall = bound > capacity ? 1u : 0u;
    c.m = c.tooSmall ? 0 : m; c.at = 0; c.cnt = 0; c.out = 0;
}

// The part after the current one, of at most P chunks; packedEnd: where the current part's frames end in the output (unused before the
// first part).  Returns whether there is such a part.
ZB_HD bool citem_advance(CItemCursor& c, u32 P, u64 packedEnd) {
    if (c.cnt) c.out = packedEnd;
    c.at += c.cnt;
    u64 const left = c.m - c.at;
    c.cnt = (u32)(left < P ? left : P);
    return c.cnt != 0;
}

// The item of chunk j < m: the last i with first[i] <= j (every item has at least one chunk, so first is strictly increasing).
ZB_HD u32 citem_of(const u64* first, u32 n, u64 j) {
    u32 lo = 0, hi = n - 1;
    while (lo < hi) {
        u32 const mid = (lo + hi + 1) >> 1;
        if (first[mid] <= j) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// Boundary k (0 ... P) of the part: slot k's input is [boundary k, boundary k + 1), an offset into the call's input.  The slots past the
// part's chunks are empty at the end of its last chunk.  *item: the item of slot k's chunk (k < cnt).
ZB_HD u64 citem_boundary(const CItemCursor& c, u32 k, u32* item) {
    u64 const j = c.at + (k < c.cnt ? k : c.cnt);
    if (j >= c.m) return c.srcOff[c.n];
    u32 const i = citem_of(c.first, c.n, j);
    *item = i;
    return c.srcOff[i] + (j - c.first[i]) * c.chunkSize;
}

// What slot k's frame result r counts as in the packing: r for a chunk of the part; an error, so that it is neither scanned nor packed,
// for a padding slot.
ZB_HD u64 citem_slot_size(const CItemCursor& c, u32 k, u64 r) { return k < c.cnt ? r : (u64)ERR(E_GENERIC); }

// What slot k's frame result r packs as: the frame, and after the last chunk of its item that item's table of T bytes.
ZB_HD u64 citem_slot_room(u64 r, bool last, u64 T) { return isErr((size_t)r) || !last ? r : r + T; }

// The key of chunk j's frame result r: its error code after its position, so that an item's least key is its first error; ~0 for a size.
ZB_HD u64 citem_error_key(u64 j, u64 r) { return isErr((size_t)r) ? (j << 8) | (u64)(0 - r) : ~0ull; }

// Item i's result once every part has run: the sum of its frames' sizes, or the code of its least key, or dstSize_tooSmall.
ZB_HD u64 citem_result(const CItemCursor& c, u64 sum, u64 key) {
    return c.tooSmall ? (u64)ERR(E_dstSize_tooSmall) : key == ~0ull ? sum : (u64)ERR((int)(key & 0xFF));
}

// The bytes chunk jj of an item of `size` bytes holds.
ZB_HD u64 citem_chunk_len(u64 size, u64 chunkSize, u64 jj) { u64 const at = jj * chunkSize; return size - at < chunkSize ? size - at : chunkSize; }

// Once the results are final: the table entry of chunk j < m, whose frame's size is csize and checksum xxh (its last four bytes), in the
// table after item i's frames -- which ends where item i + 1 starts.  An item that failed has no table.
ZB_HD void citem_table_entry(const CItemCursor& c, u64 j, u32 csize, u32 xxh) {
    u32 const i = citem_of(c.first, c.n, j);
    if (isErr((size_t)c.results[i])) return;
    u64 const k = c.first[i + 1] - c.first[i], jj = j - c.first[i];
    u8* const t = c.dst + c.dstOff[i + 1] - citem_table_size(k, c.E);
    seek_write_entry(t + SEEK_HEADER + jj * c.E, csize, (u32)citem_chunk_len(c.srcOff[i + 1] - c.srcOff[i], c.chunkSize, jj), xxh, c.E);
}
// The header and footer of item i's table.
ZB_HD void citem_table_ends(const CItemCursor& c, u32 i) {
    if (isErr((size_t)c.results[i])) return;
    u64 const k = c.first[i + 1] - c.first[i];
    seek_write_header(c.dst + c.dstOff[i + 1] - citem_table_size(k, c.E), k, c.E);
    seek_write_footer(c.dst + c.dstOff[i + 1], k, c.E);
}

}  // namespace zb
