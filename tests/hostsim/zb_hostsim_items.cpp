// zb_hostsim_items.cpp -- TEST-ONLY: the pieces of the decoder's source (zstd_jni_b200/csrc/*.cuh) that decode an item frame by frame
// and verify checksums on the staged decoder: item_walk and the decode list built on it (zb_decode_list.cuh), xxh64_warp on the 32-lane
// emulator (simt_emu.h), and dec_prepare's verdict.
// tests/test_multiframe_items.py compiles it; it is never loaded by the product path.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include "../../zstd_jni_b200/csrc/zb_decode.cuh"
#include "../../zstd_jni_b200/csrc/zb_decode_fast.cuh"
#include "../../zstd_jni_b200/csrc/zb_decode_list.cuh"
#include "simt_emu.h"

extern "C" {

// item_walk over src (copied with slack on both sides, as the kernels' loads need): the number of frames walked; out7 receives up to
// outMax records {srcOff, srcSize, contentSize, nBlocks, checksum, hasContentSize, skippable}; *split = the item may be split.
unsigned zbi_item_walk(const void* src, size_t size, unsigned long long capacity, unsigned long long* out7, unsigned outMax, int* split) {
    using namespace zb;
    u8* in = (u8*)calloc(1, size + 64);
    memcpy(in + 16, src, size);
    ItemFrame* fr = (ItemFrame*)calloc(outMax ? outMax : 1, sizeof(ItemFrame));
    bool ok = false;
    u32 const n = item_walk(in + 16, size, capacity, fr, outMax, &ok);
    for (u32 k = 0; k < n && k < outMax; k++) {
        unsigned long long* const o = out7 + 7 * k;
        o[0] = fr[k].srcOff; o[1] = fr[k].srcSize; o[2] = fr[k].contentSize; o[3] = fr[k].nBlocks; o[4] = fr[k].checksum;
        o[5] = fr[k].hasContentSize; o[6] = fr[k].skippable;
    }
    *split = ok ? 1 : 0;
    free(in); free(fr);
    return n;
}

// XXH64 of p[0, len) placed `offset` bytes past a 16-byte boundary: serial (lanes = 1) or xxh64_warp on an emulated group of `lanes`
// lanes (4, 8, 16 or 32), every lane of which must return the same value (else 0 with *uniform = 0).
unsigned long long zbi_xxh64(const void* p, size_t len, int offset, int lanes, int* uniform) {
    using namespace zb;
    u8* in = (u8*)aligned_alloc(16, (len + 96) / 16 * 16);
    memset(in, 0xA5, (len + 96) / 16 * 16);
    memcpy(in + 16 + offset, p, len);
    const u8* const q = in + 16 + offset;
    u64 h[32]; int n = 1;
    *uniform = 1;
    if (lanes == 32) { run_warp<32>([&](const WarpEmuT<32>& w) { h[w.lane] = xxh64_warp(w, q, len); }); n = 32; }
    else if (lanes == 16) { run_warp<16>([&](const WarpEmuT<16>& w) { h[w.lane] = xxh64_warp(w, q, len); }); n = 16; }
    else if (lanes == 8) { run_warp<8>([&](const WarpEmuT<8>& w) { h[w.lane] = xxh64_warp(w, q, len); }); n = 8; }
    else if (lanes == 4) { run_warp<4>([&](const WarpEmuT<4>& w) { h[w.lane] = xxh64_warp(w, q, len); }); n = 4; }
    else h[0] = xxh64(q, len);
    for (int i = 1; i < n; i++) if (h[i] != h[0]) *uniform = 0;
    u64 const r = *uniform ? h[0] : 0;
    free(in);
    return r;
}

// dec_prepare's verdict on one item: the descriptor's mode (0: the fused kernel decodes the item).
unsigned zbi_staged_mode(const void* src, size_t size, size_t dstCapacity) {
    using namespace zb;
    DecShared* S = (DecShared*)calloc(1, sizeof(DecShared));
    u8* in = (u8*)calloc(1, size + 64);
    memcpy(in + 16, src, size);
    u16* huf = (u16*)calloc(FAST_HUF_ENTRIES, 2);
    u32* fse = (u32*)calloc(FAST_FSE_ENTRIES, 4);
    DecDesc d;
    WarpHost w; dec_prepare(w, *S, in + 16, size, dstCapacity, &d, huf, fse);
    free(S); free(in); free(huf); free(fse);
    return d.mode;
}

// plan_decode_list over n items back to back at src (input offsets srcOff, output offsets dstOff, n + 1 each), the workspace reservation
// answering reserveOk.  Returns the number of entries; split[i] = item i was cut, eSrc / eDst = the entries' offsets (up to eMax + 1 of
// each), *asked = how often the reservation was asked (and the entry count it was asked for in *askedFor).
size_t zbi_decode_list(const void* src, const unsigned long long* srcOff, const unsigned long long* dstOff, size_t n, int reserveOk,
                       unsigned char* split, unsigned long long* eSrc, unsigned long long* eDst, size_t eMax, int* asked, size_t* askedFor) {
    using namespace zb;
    size_t const total = (size_t)srcOff[n];
    u8* in = (u8*)calloc(1, total + 64);
    memcpy(in + 16, src, total);
    std::vector<u64> so(srcOff, srcOff + n + 1), dof(dstOff, dstOff + n + 1);
    DecodeList L;
    *asked = 0; *askedFor = 0;
    plan_decode_list(L, n, in + 16, so.data(), dof.data(), true, [&](size_t m) { ++*asked; *askedFor = m; return reserveOk != 0; });
    for (size_t i = 0; i < n; i++) split[i] = L.split[i];
    for (size_t j = 0; j <= L.m && j <= eMax; j++) { eSrc[j] = L.src[j]; eDst[j] = L.dst[j]; }
    free(in);
    return L.m;
}

}
