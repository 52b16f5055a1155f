// zb_hostsim_opt.cpp -- TEST-ONLY host instantiation of the encoder with the optimal parser's workspace
// (enc_opt_work_carve), so that `pytest -m "not gpu"` runs levels 13..22 and strategies btopt ... btultra2 on the
// very source the CUDA kernels are built from.  Never loaded by the product path.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include "../../zstd_jni_b200/csrc/zb_encode.cuh"
#include "simt_emu.h"

extern "C" {

// ov7 = {windowLog, chainLog, hashLog, searchLog, minMatch, targetLength, strategy} (0 = from the level) or NULL.
// emu != 0: both stages on the emulated 32-lane warp; otherwise one lane.
size_t zbo_compress(void* dst, size_t dstCapacity, const void* src, size_t srcSize, int level, unsigned flags, const unsigned* ov7, int emu) {
    using namespace zb;
    if (srcSize > BLOCKSIZE_MAX) return ERR(E_srcSize_wrong);
    CParams ov = { 0, 0, 0, 0, 0, 0, 0 };
    if (ov7) ov = CParams{ ov7[0], ov7[1], ov7[2], ov7[3], ov7[4], ov7[5], ov7[6] };
    const CParams* const ovp = ov.any_set() ? &ov : nullptr;
    EncShared* S = (EncShared*)calloc(1, sizeof(EncShared));
    u8* wk = (u8*)calloc(1, enc_work_bytes() + 64);
    u8* wo = (u8*)malloc(enc_opt_work_bytes());
    memset(wo, 0xA5, enc_opt_work_bytes());       // the reference does not clear this workspace either: nothing may depend on it
    EncWork W = enc_work_carve(wk);
    enc_opt_work_carve(W, wo);
    size_t const bound = compress_bound(srcSize);
    u8* slot = (u8*)calloc(1, bound + 64);
    u8* in = (u8*)calloc(1, srcSize + 64);
    memcpy(in + 16, src, srcSize);
    size_t r;
    if (emu) {
        size_t results[32]; u32 nbSeqs[32], lastLLs[32];
        run_warp<32>([&](const WarpEmuT<32>& w) { results[w.lane] = parse_stage(w, W, in + 16, srcSize, level, &nbSeqs[w.lane], &lastLLs[w.lane], ovp); });
        r = results[0];
        for (int i = 1; i < 32; i++) if (results[i] != r || nbSeqs[i] != nbSeqs[0] || lastLLs[i] != lastLLs[0]) r = ERR(E_GENERIC);
        if (!isErr(r)) {
            run_warp<32>([&](const WarpEmuT<32>& w) { results[w.lane] = encode_stage(w, *S, W, slot, bound < 18 ? 18 : bound, in + 16, srcSize, level, nbSeqs[0], lastLLs[0], flags, ovp); });
            r = results[0];
            for (int i = 1; i < 32; i++) if (results[i] != r) r = ERR(E_GENERIC);
        }
    } else {
        WarpHost w;
        r = compress_frame(w, *S, W, slot, bound < 18 ? 18 : bound, in + 16, srcSize, level, flags, ovp);
    }
    if (!isErr(r)) { if (r > dstCapacity) r = ERR(E_dstSize_tooSmall); else memcpy(dst, slot, r); }
    free(S); free(wk); free(wo); free(slot); free(in);
    return r;
}

}
