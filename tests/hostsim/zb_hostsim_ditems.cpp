// zb_hostsim_ditems.cpp -- TEST-ONLY host instantiation of the plan of zstdb200_decompress_items_device and zstdb200_decompress_bound_device
// (zstd_jni_b200/csrc/zb_decompress_items.cuh): every item's bound, the saturating scan of the rooms in k_ditem_scan's grouping (1024
// threads, 32 lanes a warp), the fit check, the offsets the decoders run on and the results.  The decoders' results are stand-ins the
// caller gives per item.  tests/test_device_decompress_items.py compiles it; it is never loaded by the product path.
#include <vector>
#include "../../zstd_jni_b200/csrc/zb_decompress_items.cuh"

using namespace zb;

namespace {
// k_ditem_scan: each of 1024 threads sums its run of items, the 32 lanes of each warp and then the 32 warps are scanned as the shuffles
// do (lane l adds lane l - o for o = 1, 2, 4 ...), and every thread writes its run's offsets from the sum before it.
void scan_rooms(const u64* bounds, u64* offsets, u32 n) {
    constexpr u32 T = 1024;
    u32 const per = (n + T - 1) / T;
    std::vector<u64> local(T, 0), v(T);
    for (u32 t = 0; t < T; t++)
        for (u32 i = t * per; i < t * per + per && i < n; i++) local[t] = sat_add(local[t], ditem_room(bounds[i]));
    auto shuffle_scan = [](u64* x, u32 lanes) {
        for (u32 o = 1; o < lanes; o <<= 1) {
            std::vector<u64> const before(x, x + lanes);
            for (u32 l = o; l < lanes; l++) x[l] = sat_add(before[l - o], before[l]);
        }
    };
    v = local;
    for (u32 w = 0; w < T / 32; w++) shuffle_scan(v.data() + 32 * w, 32);
    u64 warpSum[32];
    for (u32 w = 0; w < 32; w++) warpSum[w] = v[32 * w + 31];
    shuffle_scan(warpSum, 32);
    for (u32 t = 0; t < T; t++) {
        u64 base = sat_add(t >> 5 ? warpSum[(t >> 5) - 1] : 0, t & 31 ? v[t - 1] : 0);
        for (u32 i = t * per; i < t * per + per && i < n; i++) { offsets[i] = base; base = sat_add(base, ditem_room(bounds[i])); }
    }
    offsets[n] = warpSum[31];
}
}  // namespace

extern "C" {

// ditem_bound of src[0, size).
unsigned long long zbd_bound(const unsigned char* src, size_t size, unsigned magicless) { return ditem_bound(src, size, magicless); }

// The plan of n items of the given bounds for an output of `capacity` bytes: dstOff (n + 1) as k_ditem_scan writes it, the input and
// output offsets the decoders run on (runSrc, runDst: n + 1 each, from srcOff and dstOff as k_ditem_fit picks them) and every item's
// result after k_ditem_finish, the decoders having given decoded[i].  Returns whether the rooms fit.
int zbd_plan(const unsigned long long* bounds, size_t n, unsigned long long capacity, const unsigned long long* srcOff,
             const unsigned long long* decoded, unsigned long long* dstOff, unsigned long long* runSrc, unsigned long long* runDst,
             unsigned long long* results) {
    scan_rooms((const u64*)bounds, (u64*)dstOff, (u32)n);
    bool const fits = ditem_fits(dstOff[n], capacity);
    for (size_t i = 0; i <= n; i++) { runSrc[i] = fits ? srcOff[i] : 0; runDst[i] = fits ? dstOff[i] : 0; }
    for (size_t i = 0; i < n; i++) results[i] = ditem_result(fits, decoded[i]);
    return fits;
}

}
