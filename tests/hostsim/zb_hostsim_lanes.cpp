// zb_hostsim_lanes.cpp -- TEST-ONLY: the compressor's kernel source (zstd_jni_b200/csrc/zb_encode.cuh) as the CUDA build runs it
// with parse_lanes = 4, 8, 16 or 32: stage 1 (k_parse) on an emulated group of that many lanes, stage 2 (k_entropy) on a 32-lane
// warp (simt_emu.h).  tests/test_parse_geometry.py compiles it; it is never loaded by the product path.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include "../../zstd_jni_b200/csrc/zb_encode.cuh"
#include "simt_emu.h"

// Stage 1 on one emulated group of LANES lanes; every lane must return the same result, nbSeq and lastLL.
template <int LANES>
static size_t emu_parse(const zb::EncWork& W, const zb::u8* src, size_t srcSize, int level, const zb::CParams* ov, zb::u32* nbSeq, zb::u32* lastLL) {
    using namespace zb;
    size_t results[LANES]; u32 nbSeqs[LANES], lastLLs[LANES];
    run_warp<LANES>([&](const WarpEmuT<LANES>& w) { results[w.lane] = parse_stage(w, W, src, srcSize, level, &nbSeqs[w.lane], &lastLLs[w.lane], ov); });
    size_t r = results[0];
    for (int i = 1; i < LANES; i++) if (results[i] != r || nbSeqs[i] != nbSeqs[0] || lastLLs[i] != lastLLs[0]) r = ERR(E_GENERIC);
    *nbSeq = nbSeqs[0]; *lastLL = lastLLs[0];
    return r;
}

extern "C" {

// ov7 = {windowLog, chainLog, hashLog, searchLog, minMatch, targetLength, strategy} (0 = from the level; null: all from the level);
// flags as for zbh_compress_flags.  Frame size or error code.
size_t zbl_compress(void* dst, size_t dstCapacity, const void* src, size_t srcSize, int level, unsigned flags, const unsigned* ov7, int lanes) {
    using namespace zb;
    if (srcSize > BLOCKSIZE_MAX) return ERR(E_srcSize_wrong);
    if (lanes != 4 && lanes != 8 && lanes != 16 && lanes != 32) return ERR(E_parameter_unsupported);
    CParams ov = { 0, 0, 0, 0, 0, 0, 0 };
    if (ov7) ov = { ov7[0], ov7[1], ov7[2], ov7[3], ov7[4], ov7[5], ov7[6] };
    const CParams* const ovp = ov.any_set() ? &ov : nullptr;
    EncShared* S = (EncShared*)calloc(1, sizeof(EncShared));
    u8* wk = (u8*)calloc(1, enc_work_bytes() + 64);
    EncWork W = enc_work_carve(wk);
    size_t const bound = compress_bound(srcSize);
    u8* slot = (u8*)calloc(1, bound + 64);
    // inputs are read with aligned 8-byte loads: give the copy slack on both sides
    u8* in = (u8*)calloc(1, srcSize + 64);
    memcpy(in + 16, src, srcSize);
    u32 nbSeq = 0, lastLL = 0;
    size_t r = lanes == 4 ? emu_parse<4>(W, in + 16, srcSize, level, ovp, &nbSeq, &lastLL)
             : lanes == 8 ? emu_parse<8>(W, in + 16, srcSize, level, ovp, &nbSeq, &lastLL)
             : lanes == 16 ? emu_parse<16>(W, in + 16, srcSize, level, ovp, &nbSeq, &lastLL)
             : emu_parse<32>(W, in + 16, srcSize, level, ovp, &nbSeq, &lastLL);
    if (!isErr(r)) {
        size_t results[32];
        run_warp<32>([&](const WarpEmuT<32>& w) { results[w.lane] = encode_stage(w, *S, W, slot, bound < 18 ? 18 : bound, in + 16, srcSize, level, nbSeq, lastLL, flags, ovp); });
        r = results[0];
        for (int i = 1; i < 32; i++) if (results[i] != r) r = ERR(E_GENERIC);   // the return value must be warp-uniform
    }
    if (!isErr(r)) { if (r > dstCapacity) r = ERR(E_dstSize_tooSmall); else memcpy(dst, slot, r); }
    free(S); free(wk); free(slot); free(in);
    return r;
}

}
