// zb_hostsim_stream.cpp -- TEST-ONLY host instantiation of a streamed frame (zstdb200_fstream_*, zb_decode_segment.cuh): segments decoded
// from their own staged copy of the input, the history in a ring of a power-of-two size, and the fused decoder's resume entry from any
// block boundary on.  Never loaded by the product path.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>
#include "../../zstd_jni_b200/csrc/zb_decode_segment.cuh"

using namespace zb;

extern "C" {

// One frame in segments of segBlocks blocks, also cut at block resumeFrom: the segments before it on the segment decoder, whose copies
// before the segment read a ring of 2^ringLog bytes (0: the least power of two that holds the window and one segment), the blocks from
// it on through seg_resume with the whole frame so far as history and the caller's capacity (stream = 0), or as the frame stream runs
// it (stream = 1): the last window copied out of the ring as history, room for any segment, and the block headers the reference's
// streaming decoder rejects refused before their segment.  Each segment is decoded from a copy of its blocks only, which is
// overwritten once the segment is done.  *status: 0 decoded (returns the size), 1 an error code (returned), 2 the segment decoder
// could not vouch for a segment.
size_t zbst_decode(void* dst, size_t cap, const void* src, size_t size, unsigned segBlocks, unsigned resumeFrom, unsigned ringLog, int stream,
                   int* status) {
    const u8* const frame = (const u8*)src;
    FrameHeader fh; u32 xxh = 0;
    u32 const n = frame_walk(frame, size, &fh, 0xFFFFFFFFu, nullptr, &xxh);
    *status = 2;
    if (!n) return 0;
    std::vector<u64> refs(n);
    frame_walk(frame, size, &fh, 0xFFFFFFFFu, refs.data(), &xxh);
    u32 const B = segBlocks ? segBlocks : n;
    size_t const segOut = (size_t)B * (fh.blockSizeMax + LIT_MARGIN);
    u64 R = 1;
    if (ringLog) R <<= ringLog; else while (R < fh.windowSize + segOut) R <<= 1;
    std::vector<u8> ring((size_t)R), lin(cap + 2 * (size_t)fh.blockSizeMax + segOut + 256), scratch(BLOCKSIZE_MAX + 256);
    constexpr size_t LS = BLOCKSIZE_MAX + 64;
    std::vector<SegBlock> blocks(B);
    std::vector<u16> huf((size_t)B * SEG_HUF_ENTRIES);
    std::vector<u32> fse((size_t)B * FAST_FSE_ENTRIES), offs((size_t)B * FAST_MAXS), link((size_t)B * BLOCKSIZE_MAX);
    std::vector<u8> lit((size_t)B * LS);
    std::vector<u64> seqs((size_t)B * FAST_MAXS);
    SegCarry* c = (SegCarry*)calloc(1, sizeof(SegCarry));
    DecShared* S = (DecShared*)calloc(1, sizeof(DecShared));
    seg_carry_init(c, ~0ull);
    WarpHost h;
    size_t result = 0, headerError = 0;
    std::vector<u8> hist;
    for (u32 first = 0; first < n;) {
        u32 cnt = n - first < B ? n - first : B;
        if (first < resumeFrom && first + cnt > resumeFrom) cnt = resumeFrom - first;
        if (stream)
            for (u32 j = 0; j < cnt; j++)
                if (stream_block_error((u32)(refs[first + j] >> 32), fh.blockSizeMax)) { cnt = j; headerError = ERR(E_corruption_detected); break; }
        if (cnt == 0) { *status = 1; result = headerError; break; }
        // the segment's own copy of its blocks
        std::vector<u8> in;
        std::vector<u64> r(cnt);
        for (u32 j = 0; j < cnt; j++) {
            u32 const off = (u32)refs[first + j], bh = (u32)(refs[first + j] >> 32), cs = ((bh >> 1) & 3) == 1 ? 1 : bh >> 3;
            r[j] = (u64)in.size() | ((u64)bh << 32);
            in.insert(in.end(), frame + off, frame + off + 3 + cs);
        }
        in.resize(in.size() + 64);
        u64 const start = c->pos;
        if (first >= resumeFrom) {
            if (lin.size() < start + segOut + 2 * (size_t)fh.blockSizeMax + 256) lin.resize(start + segOut + 2 * (size_t)fh.blockSizeMax + 256);
            size_t const room = segOut + 2 * (size_t)fh.blockSizeMax + 128, left = start < cap ? (size_t)(cap - start) : 0;
            size_t got;
            if (stream) {          // the last window out of the ring, right before the segment's room
                size_t const hl = (size_t)(start < fh.windowSize ? start : fh.windowSize);
                hist.assign(hl + room + 64, 0);
                for (size_t p = 0; p < hl; p++) hist[p] = ring[(start - hl + p) & (R - 1)];
                got = stream_resume_result(seg_resume(h, *S, in.data(), r.data(), cnt, fh.blockSizeMax, hist.data(), hist.data() + hl, room,
                                                      scratch.data(), c));
                if (!isErr(got)) memcpy(lin.data() + start, hist.data() + hl, got);
            } else         // the caller's capacity, as the whole-frame decode has it
                got = seg_resume(h, *S, in.data(), r.data(), cnt, fh.blockSizeMax, lin.data(), lin.data() + start, left < room ? left : room,
                                 scratch.data(), c);
            if (isErr(got)) { *status = 1; result = got; break; }
            for (size_t p = 0; p < got; p++) ring[(start + p) & (R - 1)] = lin[start + p];
        } else {
            for (u32 j = 0; j < cnt; j++)
                seg_prepare(h, *S, in.data(), (u32)r[j], (u32)(r[j] >> 32), fh.blockSizeMax, &blocks[j], &huf[(size_t)j * SEG_HUF_ENTRIES],
                            &fse[(size_t)j * FAST_FSE_ENTRIES]);
            seg_tables(blocks.data(), cnt, c, false, ~0ull);
            if (!c->bad) {
                for (u32 j = 0; j < cnt; j++) for (int k = 0; k < 4; k++) seg_huf(blocks.data(), j, k, in.data(), huf.data(), c, &lit[(size_t)j * LS]);
                for (u32 j = 0; j < cnt; j++) seg_seq(blocks.data(), j, in.data(), fse.data(), c, &seqs[(size_t)j * FAST_MAXS], &offs[(size_t)j * FAST_MAXS]);
                seg_scan(blocks.data(), cnt, c, fh.blockSizeMax);
            }
            if (!c->bad) {
                for (u32 j = 0; j < cnt; j++) seg_offsets(blocks.data(), j, &seqs[(size_t)j * FAST_MAXS], &offs[(size_t)j * FAST_MAXS]);
                seg_carry_tables(h, blocks.data(), huf.data(), fse.data(), c);
                SegRec Rec[1];
                for (u32 j = 0; j < cnt; j++)
                    seg_fill(h, Rec, blocks.data(), j, in.data(), &lit[(size_t)j * LS], &seqs[(size_t)j * FAST_MAXS], &offs[(size_t)j * FAST_MAXS],
                             ring.data(), R - 1, fh.windowSize, start, link.data(), c);
            }
            if (c->bad) break;
            for (u64 p = 0; p < c->pos - start; p++) ring[(start + p) & (R - 1)] = seg_jump(link.data(), (u32)p);
            if (lin.size() < c->pos) lin.resize(c->pos + 256);
            for (u64 p = start; p < c->pos; p++) lin[p] = ring[p & (R - 1)];
        }
        memset(in.data(), 0xA5, in.size());          // nothing may read the segment's input after it
        first += cnt;
        if (headerError) { *status = 1; result = headerError; break; }
    }
    if (*status == 2 && !c->bad) {
        if (fh.hasContentSize && c->pos != fh.contentSize) { *status = 1; result = ERR(E_corruption_detected); }
        else if (fh.checksum && (u32)xxh64(lin.data(), (size_t)c->pos) != xxh) { *status = 1; result = ERR(E_checksum_wrong); }
        else if (c->pos > cap) { *status = 1; result = ERR(E_dstSize_tooSmall); }
        else { *status = 0; result = (size_t)c->pos; memcpy(dst, lin.data(), result); }
    }
    free(c); free(S);
    return result;
}

}
