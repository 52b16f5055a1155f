// zb_decode_ranges.cuh -- the plan of zstdb200_decompress_ranges_device: byte ranges of items in device memory regenerated from the
// frames that hold them, located on the GPU.  The kernels k_range_* in zb_capi.cu are thin wrappers of these functions;
// tests/hostsim/zb_hostsim_ranges.cpp runs them on the host.
//
// Request r asks for the bytes [b, e) of one item's regenerated content.  Its frames are found by a walk from the item's start
// (range_next over frame_size_info): every zstd frame passed declares its content size, so the walk knows where each frame's bytes sit
// without decoding it.  A frame is an entry of the request when it regenerates at least one byte of [b, e).  range_locate walks each
// request as far as e, counts its entries and those covered only in part, keeps a cursor at its first entry, the bytes it will return,
// and the first error met (as a (position, code) key, range_key).  The counts are scanned into each request's first entry and first
// partial entry.  Then the entries are decoded in parts of at most P entries, of which at most S are covered in part (range_part): every
// request with entries in the part continues its walk from its cursor and writes their slots (range_slot) -- straight into its output
// for a frame it covers wholly, into a 128 KB scratch slot for one it covers in part.  Once decoded, each slot's result settles into its
// request (range_entry_key) and a partial slot's slice is copied out.  A request's result is its least key's code, or its bytes
// (range_result).
//
// With seek tables, a request whose item ends with a valid table (seek_table_read, and entries whose compressed sizes sum to the bytes
// before it) is located through the table instead (range_locate_seek): a group of lanes scans the entries W at a time with prefix sums of
// their sizes, counts the entries that hold a byte of [b, e) -- entries of regenerated size 0 are passed -- and keeps a cursor of entry
// index, input offset and content offset, from which range_fill_seek reaches every later entry in O(1).  Each entry's frame must pass
// seek_frame_check, regenerate exactly the entry's size, and with table checksums hash to the entry's (range_entry_verify).  An item
// without a valid table is walked as above.
#pragma once
#include "zb_decompress_items.cuh"
#include "zb_seek_table.cuh"

namespace zb {

constexpr u64 RANGE_PARTIAL_MAX = BLOCKSIZE_MAX;      // largest frame a range may cover in part: the size of a scratch slot
constexpr u32 NO_SCRATCH = 0xFFFFFFFFu;

// A point of a request's walk: the input offset of the next frame in its item and the content offset where that frame's bytes start.
struct RangeWalk { u64 pos, at; };
// A frame the walk found: its input offset and compressed size, its content offset and content size.
struct RangeFrame { u64 pos, size, at, cs; };
// What range_locate leaves for the parts: the walk at the request's next entry, its least error key (~0: none), and which of its
// entries are covered in part -- bit 0 the first, bit 1 the last (a request of one entry uses bit 0 alone); bit 2 (RANGE_SEEK) when
// the request is located through its item's seek table, whose entry `entry` the walk is at.
struct RangeReq { RangeWalk cur; u64 err; u32 flags, entry; };
constexpr u32 RANGE_SEEK = 4;

// The key of an error `code` met at input offset pos of the item: the least key is the first error in item order (citem_error_key's
// order).  Input offsets stay far below 2^56.
ZB_HD u64 range_key(u64 pos, size_t code) { return (pos << 8) | (u64)(0 - code); }

// The next frame of item src[0, size) that regenerates a byte of [b, e), the walk going on from w: skippable frames, empty frames and
// frames that end at or before b are passed.  Returns 1 with the frame in *f and w past it; 0 when the walk reaches e or the item's end
// first; or the error that stops the walk, w left at the frame that gives it: frame_size_info's, or parameter_unsupported for a zstd
// frame that declares no content size, or one larger than RANGE_PARTIAL_MAX that [b, e) covers only in part.
ZB_HDN size_t range_next(const u8* src, size_t size, u32 magicless, u64 b, u64 e, RangeWalk& w, RangeFrame* f) {
    while (w.pos < size && w.at < e) {
        FrameHeader fh; u64 blocks;
        size_t const fs = frame_size_info(src + w.pos, (size_t)(size - w.pos), magicless, &fh, &blocks);
        if (isErr(fs)) return fs;
        if (fh.skippable) { w.pos += fs; continue; }
        if (!fh.hasContentSize) return ERR(E_parameter_unsupported);
        u64 const at = w.at, cs = fh.contentSize, end = sat_add(at, cs);
        if (cs == 0 || end <= b) { w.pos += fs; w.at = end; continue; }
        if ((at < b || end > e) && cs > RANGE_PARTIAL_MAX) return ERR(E_parameter_unsupported);
        f->pos = w.pos; f->size = fs; f->at = at; f->cs = cs;
        w.pos += fs; w.at = end;
        return 1;
    }
    return 0;
}

// The end of a request for len bytes at b (saturating).
ZB_HD u64 range_end(u64 b, u64 len) { return sat_add(b, len); }

// Request for [b, b + len) of `item` among n items (item i: src[srcOff[i], srcOff[i + 1])): walked as far as it reaches.  *q: the cursor
// at its first entry, its least error key and partial flags; *count its entries, *partial how many of them are covered in part, *bytes
// what it returns when no entry fails -- the bytes of [b, e) the item has (fewer when its content ends first).  An item beyond n gives
// parameter_outOfBound; an empty request reads nothing.  Entries before a walk error are kept: a decode error among them comes first.
ZB_HDN void range_locate(const u8* src, const u64* srcOff, u64 n, u64 item, u64 b, u64 len, u32 magicless, RangeReq* q, u64* count,
                         u64* partial, u64* bytes) {
    RangeReq r{};
    r.err = ~0ull;
    u64 cnt = 0, got = 0;
    if (item >= n) r.err = range_key(0, ERR(E_parameter_outOfBound));
    else if (len) {
        const u8* const s = src + srcOff[item];
        size_t const size = (size_t)(srcOff[item + 1] - srcOff[item]);
        u64 const e = range_end(b, len);
        RangeWalk w{0, 0};
        RangeFrame f;
        for (;;) {
            size_t const k = range_next(s, size, magicless, b, e, w, &f);
            if (isErr(k)) { r.err = range_key(w.pos, k); break; }
            if (k == 0) break;
            bool const part = f.at < b || f.at + f.cs > e;
            if (cnt == 0) { r.cur.pos = f.pos; r.cur.at = f.at; r.flags = part; }
            else if (part) r.flags |= 2;
            got += (f.at + f.cs < e ? f.at + f.cs : e) - (f.at > b ? f.at : b);
            cnt++;
        }
    }
    *q = r; *count = cnt; *bytes = got;
    *partial = cnt == 0 ? 0 : (u64)(r.flags & 1) + (u64)((r.flags >> 1) & 1);
}

// Whether entry j (0-based) of a request of `count` entries and partial flags `flags` is covered in part, and how many of its entries
// before j are.
ZB_HD bool range_entry_partial(u32 flags, u64 j, u64 count) { return (j == 0 && (flags & 1)) || (j + 1 == count && j > 0 && (flags & 2)); }
ZB_HD u64 range_partial_before(u32 flags, u64 j) { return j > 0 && (flags & 1) ? 1 : 0; }

// The request whose entries hold entry j of first[m] (first: m + 1 nondecreasing, j < first[m]): the last r with first[r] <= j.
ZB_HD u64 range_find(const u64* first, u64 m, u64 j) {
    u64 lo = 0, hi = m - 1;
    while (lo < hi) {
        u64 const mid = lo + (hi - lo + 1) / 2;
        if (first[mid] <= j) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// A part of the entries: [at, at + cnt), q entries covered in part before `at`, held by requests r0 .. r1.
struct RangePart { u64 at, q, r0, r1; u32 cnt; };

// The part that starts at entry `at`: at most P entries, of which at most S covered in part (first, pfirst: the scans of the m requests'
// entries and partial entries).  cnt 0: no entry is left.
ZB_HD RangePart range_part(const u64* first, const u64* pfirst, const RangeReq* req, u64 m, u64 at, u32 P, u32 S) {
    RangePart p{};
    p.at = at;
    if (m == 0 || at >= first[m]) return p;
    u64 cnt = first[m] - at < P ? first[m] - at : P;
    p.r0 = range_find(first, m, at);
    p.q = pfirst[p.r0] + range_partial_before(req[p.r0].flags, at - first[p.r0]);
    if (p.q + S < pfirst[m]) {      // the part ends before the partial entry S places on
        u64 const qq = p.q + S, rq = range_find(pfirst, m, qq);
        u64 const j = qq == pfirst[rq] && (req[rq].flags & 1) ? first[rq] : first[rq + 1] - 1;
        if (j - at < cnt) cnt = j - at;
    }
    p.cnt = (u32)cnt;
    p.r1 = range_find(first, m, at + cnt - 1);
    return p;
}

// The slot of entry f of request r ([b, e)): the frame's input [pos, pos + size) in the item, its content size cs, and where it goes.  A
// frame [b, e) covers wholly decodes straight into the request's output at `to`; one it covers in part decodes into scratch slot
// `scratch`, from which `len` bytes at `from` are copied to the request's output at `to`.  A seek-table entry's slot may carry the code
// of the check its frame failed (err, 0: none; the slot is not decoded) and the checksum its output must hash to (when `verify`).
struct RangeSlot { u64 pos, size, cs, to; u32 req, from, len, scratch, err, xxh, verify, pad; };
ZB_HD RangeSlot range_slot(const RangeFrame& f, u32 r, u64 b, u64 e, bool part, u32 scratch) {
    RangeSlot s{};
    u64 const lo = f.at > b ? f.at : b, hi = f.at + f.cs < e ? f.at + f.cs : e;
    s.pos = f.pos; s.size = f.size; s.cs = f.cs; s.req = r; s.to = lo - b;
    s.from = (u32)(lo - f.at); s.len = part ? (u32)(hi - lo) : 0; s.scratch = part ? scratch : NO_SCRATCH;
    return s;
}

// Request r's entries in part p into their slots (slots[0] is the part's first): its walk goes on from q->cur, which is left at its next
// entry.  first, last: its entries [first, last); pfirst: its first partial entry's number.  The walk was made by range_locate, so every
// frame it meets is one range_locate counted.
ZB_HD void range_fill_seek(const u8* src, size_t size, u64 b, u64 e, u32 r, u64 first, u64 last, u64 pfirst, RangeReq* q,
                            const RangePart& p, RangeSlot* slots);
ZB_HD void range_fill(const u8* src, size_t size, u32 magicless, u64 b, u64 e, u32 r, u64 first, u64 last, u64 pfirst, RangeReq* q,
                       const RangePart& p, RangeSlot* slots) {
    if (q->flags & RANGE_SEEK) { range_fill_seek(src, size, b, e, r, first, last, pfirst, q, p, slots); return; }
    u64 const j0 = first > p.at ? first : p.at, j1 = last < p.at + p.cnt ? last : p.at + p.cnt;
    RangeWalk w = q->cur;
    u32 const flags = q->flags;
    for (u64 j = j0; j < j1; j++) {
        RangeFrame f{};
        range_next(src, size, magicless, b, e, w, &f);
        bool const part = range_entry_partial(flags, j - first, last - first);
        u32 const scratch = part ? (u32)(pfirst + range_partial_before(flags, j - first) - p.q) : NO_SCRATCH;
        slots[j - p.at] = range_slot(f, r, b, e, part, scratch);
    }
    q->cur = w;
}

// The key a decoded slot's result res settles into its request: ~0 when the frame regenerated exactly its declared size, else the
// decoder's error or corruption_detected, at the frame's position.
ZB_HD u64 range_entry_key(const RangeSlot& s, u64 res) {
    if (s.err) return range_key(s.pos, ERR((int)s.err));
    if (isErr((size_t)res)) return range_key(s.pos, (size_t)res);
    return res == s.cs ? ~0ull : range_key(s.pos, ERR(E_corruption_detected));
}

// A request's result: the code of its least key, or its bytes.
ZB_HD u64 range_result(u64 err, u64 bytes) { return err == ~0ull ? bytes : (u64)ERR((size_t)(err & 0xFF)); }

// ---- through a seek table

// The check of the frame a seek-table entry lists at input offset pos of item src[0, size), csize bytes regenerating dsize: the code of
// its walk's error (frame_size_info), corruption_detected for a skippable frame, a frame of another size or one that declares another
// content size; 0 when it passes.  A frame that declares no content size passes.
ZB_HDN u32 seek_frame_check(const u8* src, size_t size, u64 pos, u32 csize, u32 dsize) {
    FrameHeader fh; u64 blocks;
    size_t const fs = frame_size_info(src + pos, (size_t)(size - pos), 0, &fh, &blocks);
    if (isErr(fs)) return (u32)(0 - fs);
    if (fh.skippable || fs != csize || (fh.hasContentSize && fh.contentSize != dsize)) return (u32)E_corruption_detected;
    return 0;
}

// The sum of v over the group's lanes, in every lane.
template <class C> ZB_HD u64 group_sum64(const C& w, u64 v) {
    for (int o = C::W / 2; o > 0; o >>= 1) v += w.shfl(v, (int)(lane_of(w) ^ (u32)o));
    return v;
}

// Request for [b, e) of item src[0, size), whose table t passed seek_table_read, located by the group w, W entries per round: prefix
// sums over the round's compressed and regenerated sizes place every entry.  An entry is the request's when it regenerates a byte of
// [b, e); one covered in part must regenerate at most RANGE_PARTIAL_MAX bytes, else the request stops there with parameter_unsupported,
// keyed by the entry's position (the entries before it kept, as range_locate keeps them).  Every entry is read, for the sum of their
// compressed sizes: false, nothing written, when it is not the bytes before the table -- the table is not valid and the item is walked.
// Else *q, *count, *partial and *bytes as range_locate leaves them, written by lane 0.
template <class C>
ZB_HD bool range_locate_seek(const C& w, const u8* src, size_t size, const SeekTable& t, u64 b, u64 e, RangeReq* q, u64* count, u64* partial,
                             u64* bytes) {
    u32 const lane = lane_of(w);
    RangeReq r{};
    r.err = ~0ull; r.flags = RANGE_SEEK;
    u64 pos = 0, at = 0, cnt = 0, got = 0;
    bool stop = false;
    for (u64 j0 = 0; j0 < t.k; j0 += (u64)C::W) {
        u64 const j = j0 + lane;
        SeekEntry x{0, 0, 0};
        if (j < t.k) x = seek_entry(src, t, j);
        u64 cs = x.csize, ds = x.dsize;
        for (int o = 1; o < C::W; o <<= 1) {      // inclusive scans
            u32 const from = lane >= (u32)o ? lane - (u32)o : lane;
            u64 const a = w.shfl(cs, (int)from), d = w.shfl(ds, (int)from);
            if (lane >= (u32)o) { cs += a; ds += d; }
        }
        u64 const epos = pos + cs - x.csize, eat = at + ds - x.dsize;      // the entry's input and content offsets
        u64 const eend = eat + x.dsize;
        bool const hit = !stop && x.dsize && eat < e && eend > b;
        bool const part = hit && (eat < b || eend > e);
        u32 hits = w.ballot(hit);
        u32 const bad = w.ballot(part && x.dsize > RANGE_PARTIAL_MAX);
        if (bad) {
            u32 const l = ctz32(bad);
            hits &= (1u << l) - 1u;
            u64 const bpos = w.shfl(epos, (int)l);
            r.err = range_key(bpos, ERR(E_parameter_unsupported));
            stop = true;
        }
        bool const mine = (hits >> lane) & 1u;
        u32 const parts = w.ballot(mine && part);
        if (hits) {
            u32 const l = ctz32(hits);
            u64 const fpos = w.shfl(epos, (int)l), fat = w.shfl(eat, (int)l);
            if (cnt == 0) {
                r.cur.pos = fpos; r.cur.at = fat; r.entry = (u32)(j0 + l); r.flags = RANGE_SEEK | ((parts >> l) & 1u);
                if (parts & ~(1u << l)) r.flags |= 2;
            } else if (parts) r.flags |= 2;
            cnt += popc32(hits);
            got += group_sum64(w, mine ? (eend < e ? eend : e) - (eat > b ? eat : b) : 0);
        }
        pos += w.shfl(cs, C::W - 1); at += w.shfl(ds, C::W - 1);
    }
    if (pos != t.at - SEEK_HEADER) return false;
    if (lane == 0) {
        *q = r; *count = cnt; *bytes = got;
        *partial = cnt == 0 ? 0 : (u64)(r.flags & 1) + (u64)((r.flags >> 1) & 1);
    }
    return true;
}

// range_locate with seek tables: an item that ends with a valid table is located through it by the group, any other walked by lane 0.
template <class C>
ZB_HD void range_locate_any(const C& w, const u8* src, const u64* srcOff, u64 n, u64 item, u64 b, u64 len, RangeReq* q, u64* count,
                            u64* partial, u64* bytes) {
    if (item < n && len) {
        const u8* const s = src + srcOff[item];
        size_t const size = (size_t)(srcOff[item + 1] - srcOff[item]);
        SeekTable t;
        if (seek_table_read(s, size, &t) && range_locate_seek(w, s, size, t, b, range_end(b, len), q, count, partial, bytes)) return;
    }
    if (lane_of(w) == 0) range_locate(src, srcOff, n, item, b, len, 0, q, count, partial, bytes);
}

// range_fill for a request located through its item's table: every entry from the cursor on, entries of regenerated size 0 passed,
// each with its frame's check and, with table checksums, the checksum its output must hash to.
ZB_HD void range_fill_seek(const u8* src, size_t size, u64 b, u64 e, u32 r, u64 first, u64 last, u64 pfirst, RangeReq* q,
                            const RangePart& p, RangeSlot* slots) {
    u64 const j0 = first > p.at ? first : p.at, j1 = last < p.at + p.cnt ? last : p.at + p.cnt;
    SeekTable t{};
    seek_table_read(src, size, &t);      // (valid: range_locate_seek located the request)
    RangeWalk w = q->cur;
    u64 k = q->entry;
    u32 const flags = q->flags;
    for (u64 j = j0; j < j1; j++) {
        SeekEntry x = seek_entry(src, t, k);
        while (x.dsize == 0) { w.pos += x.csize; x = seek_entry(src, t, ++k); }
        RangeFrame const f{w.pos, x.csize, w.at, x.dsize};
        bool const part = range_entry_partial(flags, j - first, last - first);
        u32 const scratch = part ? (u32)(pfirst + range_partial_before(flags, j - first) - p.q) : NO_SCRATCH;
        RangeSlot s = range_slot(f, r, b, e, part, scratch);
        s.err = seek_frame_check(src, size, f.pos, x.csize, x.dsize);
        s.xxh = x.xxh; s.verify = t.E == 12;
        slots[j - p.at] = s;
        w.pos += x.csize; w.at += x.dsize; k++;
    }
    q->cur = w; q->entry = (u32)k;
}

// A decoded slot's result once its output `out` is checked against its entry's checksum: checksum_wrong when the frame regenerated
// its size but the bytes hash otherwise; else res.  The group hashes together.
template <class C> ZB_HD u64 range_entry_verify(const C& w, const RangeSlot& s, u64 res, const u8* out) {
    if (!s.verify || s.err || res != s.cs) return res;
    return (u32)xxh64_warp(w, out, (size_t)s.cs) == s.xxh ? res : (u64)ERR(E_checksum_wrong);
}

}  // namespace zb
