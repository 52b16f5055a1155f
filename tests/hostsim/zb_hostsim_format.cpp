// zb_hostsim_format.cpp -- TEST-ONLY: the frame walks of the decode list and the staged decoder in either frame format, ZSTD_f_zstd1 or
// ZSTD_f_zstd1_magicless (magicless != 0), from the decoder's source (zstd_jni_b200/csrc/*.cuh).
// tests/test_decode_list_calls.py compiles it; it is never loaded by the product path.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include "../../zstd_jni_b200/csrc/zb_decode.cuh"
#include "../../zstd_jni_b200/csrc/zb_decode_fast.cuh"
#include "../../zstd_jni_b200/csrc/zb_decode_segment.cuh"

extern "C" {

// item_walk over src (copied with slack on both sides, as the kernels' loads need): the number of frames walked; out7 receives up to
// outMax records {srcOff, srcSize, contentSize, nBlocks, checksum, hasContentSize, skippable}; *split = the item may be split.
unsigned zbf_item_walk(const void* src, size_t size, unsigned long long capacity, unsigned magicless, unsigned long long* out7, unsigned outMax,
                       int* split) {
    using namespace zb;
    u8* in = (u8*)calloc(1, size + 64);
    memcpy(in + 16, src, size);
    ItemFrame* fr = (ItemFrame*)calloc(outMax ? outMax : 1, sizeof(ItemFrame));
    bool ok = false;
    u32 const n = item_walk(in + 16, size, capacity, fr, outMax, &ok, magicless);
    for (u32 k = 0; k < n && k < outMax; k++) {
        unsigned long long* const o = out7 + 7 * k;
        o[0] = fr[k].srcOff; o[1] = fr[k].srcSize; o[2] = fr[k].contentSize; o[3] = fr[k].nBlocks; o[4] = fr[k].checksum;
        o[5] = fr[k].hasContentSize; o[6] = fr[k].skippable;
    }
    *split = ok ? 1 : 0;
    free(in); free(fr);
    return n;
}

// frame_walk (seg = 0) or seg_walk (seg = 1) of an item that is one frame: the number of blocks (0: not such a frame); refs receives up
// to maxRefs block refs (offset of the block header | header << 32), *xxh the stored checksum.
unsigned zbf_frame_walk(const void* src, size_t size, unsigned magicless, int seg, unsigned long long* refs, unsigned maxRefs, unsigned* xxh) {
    using namespace zb;
    u8* in = (u8*)calloc(1, size + 64);
    memcpy(in + 16, src, size);
    FrameHeader fh; u32 x = 0;
    u32 const n = seg ? seg_walk(in + 16, size, &fh, nullptr, &x, magicless) : frame_walk(in + 16, size, &fh, 0xFFFFFFFFu, nullptr, &x, nullptr, magicless);
    if (n && n <= maxRefs) {
        u64* const r = (u64*)calloc(n, 8);
        if (seg) seg_walk(in + 16, size, &fh, r, &x, magicless); else frame_walk(in + 16, size, &fh, 0xFFFFFFFFu, r, &x, nullptr, magicless);
        for (u32 k = 0; k < n; k++) refs[k] = r[k];
        free(r);
    }
    *xxh = x;
    free(in);
    return n;
}

// The staged decoder on one item in the given format: dec_prepare, the Huffman and sequence chains, dec_exec; *mode = the descriptor's
// mode.  An item dec_prepare leaves to the fused decoder (mode 0) is decoded there, as k_decompress would.
size_t zbf_staged(void* dst, size_t dstCapacity, const void* src, size_t srcSize, unsigned magicless, unsigned* mode) {
    using namespace zb;
    DecShared* S = (DecShared*)calloc(1, sizeof(DecShared));
    u8* in = (u8*)calloc(1, srcSize + 64);
    memcpy(in + 16, src, srcSize);
    u8* out = (u8*)aligned_alloc(16, (dstCapacity + 96) / 16 * 16); memset(out, 0, (dstCapacity + 96) / 16 * 16);
    u8* lit = (u8*)calloc(1, BLOCKSIZE_MAX + 64);
    u16* huf = (u16*)calloc(FAST_HUF_ENTRIES, 2);
    u32* fse = (u32*)calloc(FAST_FSE_ENTRIES, 4);
    ExecShared* X = (ExecShared*)aligned_alloc(16, (sizeof(ExecShared) + 15) / 16 * 16);
    u64* seqs = (u64*)calloc(FAST_MAXS + 8, 8);
    DecDesc d;
    size_t r;
    {   WarpHost w; dec_prepare(w, *S, in + 16, srcSize, dstCapacity, &d, huf, fse, magicless); }
    *mode = d.mode;
    if (d.mode == 0) {
        u8* scratch = (u8*)calloc(1, BLOCKSIZE_MAX + 64);
        WarpHost w; r = decompress_item(w, *S, in + 16, srcSize, out + 16, dstCapacity, scratch, magicless);
        free(scratch);
    } else {
        const u8* blk = in + 16 + d.blockOff;
        for (int k = 0; k < 4; k++) dec_huf(&d, k, blk, huf, lit);
        dec_seq(&d, blk, fse, &h_tables, seqs);
        WarpHost w; r = dec_exec(w, *X, &d, in + 16, lit, seqs, out + 16, dstCapacity, magicless);
    }
    if (!isErr(r)) memcpy(dst, out + 16, r);
    free(S); free(in); free(out); free(lit); free(huf); free(fse); free(seqs); free(X);
    return r;
}

}
