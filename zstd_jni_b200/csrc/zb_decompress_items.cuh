// zb_decompress_items.cuh -- the plan of zstdb200_decompress_items_device / zstdb200_decompress_bound_device: every item's room in the
// output found from its own frames on the GPU, with nothing from the host.  The kernels k_ditem_* in zb_capi.cu are thin wrappers of these
// functions; tests/hostsim/zb_hostsim_ditems.cpp runs them on the host.
//
// Each item is walked frame by frame (ditem_bound: the reference's ZSTD_decompressBound); its room is that bound, or nothing when the walk
// fails (ditem_room).  The rooms are scanned with a sum that saturates (sat_add) into the output offsets, and the last offset is checked
// against the capacity (ditem_fits).  When the output is short, every item decodes from and into nothing, and then reports
// dstSize_tooSmall (ditem_result).
#pragma once
#include "zb_decode.cuh"

namespace zb {

constexpr u64 CONTENTSIZE_UNKNOWN = ~0ull, CONTENTSIZE_ERROR = ~0ull - 1;      // ZSTD_CONTENTSIZE_UNKNOWN / ZSTD_CONTENTSIZE_ERROR

// ZSTD_findFrameSizeInfo (N/decompress/zstd_decompress.c:734-799) of the frame that starts src[0, size): its header to *fh, its blocks to
// *blocks (0 for a skippable frame); returns its compressed size, or the error ZSTD_findFrameCompressedSize gives for it.  Frames of any
// size are walked.  In the magicless format there are no skippable frames (the reference's ZSTD_f_zstd1_magicless walk).
ZB_HDN size_t frame_size_info(const u8* src, size_t size, u32 magicless, FrameHeader* fh, u64* blocks) {
    *blocks = 0;
    {   size_t const r = read_frame_header(fh, src, size, magicless);
        if (r != 0) return isErr(r) ? r : ERR(E_srcSize_wrong); }      // an error, or a header cut short
    if (fh->skippable) {      // readSkippableFrameSize: a length whose frame size wraps 32 bits is refused
        if (fh->skipLen > 0xFFFFFFF7u) return ERR(E_frameParameter_unsupported);
        if ((u64)fh->skipLen + 8 > size) return ERR(E_srcSize_wrong);
        return 8 + (size_t)fh->skipLen;
    }
    size_t p = fh->headerSize;
    for (;;) {      // ZSTD_getcBlockSize, then the block inside the input
        if (size - p < 3) return ERR(E_srcSize_wrong);
        u32 const bh = load24(src + p), type = (bh >> 1) & 3;
        size_t const cSize = type == 1 ? 1 : bh >> 3;
        if (type == 3) return ERR(E_corruption_detected);
        if (cSize > size - p - 3) return ERR(E_srcSize_wrong);
        p += 3 + cSize; ++*blocks;
        if (bh & 1) break;
    }
    if (fh->checksum) {
        if (size - p < 4) return ERR(E_srcSize_wrong);
        p += 4;
    }
    return p;
}

// ZSTD_decompressBound of item src[0, size) (N/decompress/zstd_decompress.c:734-836): the sum over its frames (frame_size_info) of the
// declared content size, or, for a frame that declares none, its blocks times its largest block; skippable frames count nothing;
// CONTENTSIZE_ERROR when the item is not a whole number of frames whose headers read.  As in the reference, a declared size of
// CONTENTSIZE_UNKNOWN counts as none, one of CONTENTSIZE_ERROR is an error, and the sum wraps.
ZB_HDN u64 ditem_bound(const u8* src, size_t size, u32 magicless) {
    u64 bound = 0;
    size_t pos = 0;
    while (pos < size) {
        FrameHeader fh; u64 blocks;
        size_t const fs = frame_size_info(src + pos, size - pos, magicless, &fh, &blocks);
        if (isErr(fs)) return CONTENTSIZE_ERROR;
        pos += fs;
        if (fh.skippable) continue;
        u64 const declared = fh.hasContentSize ? fh.contentSize : CONTENTSIZE_UNKNOWN;
        if (declared == CONTENTSIZE_ERROR) return CONTENTSIZE_ERROR;
        bound += declared != CONTENTSIZE_UNKNOWN ? declared : blocks * fh.blockSizeMax;
    }
    return bound;
}

// The room of an item of bound b in the output: b, or nothing for an item that is not a whole number of frames.
ZB_HD u64 ditem_room(u64 b) { return b == CONTENTSIZE_ERROR ? 0 : b; }

// a + b, or 2^64 - 1 when that wraps (an associative sum: the scan of the rooms may add them in any grouping).
ZB_HD u64 sat_add(u64 a, u64 b) { return a + b < a ? ~0ull : a + b; }

// Whether the rooms, `total` bytes in all, fit an output of `capacity` bytes.
ZB_HD bool ditem_fits(u64 total, u64 capacity) { return total <= capacity; }

// Item i's result once decoded: the decoders' r when the rooms fit, else dstSize_tooSmall.
ZB_HD u64 ditem_result(bool fits, u64 r) { return fits ? r : (u64)ERR(E_dstSize_tooSmall); }

}  // namespace zb
