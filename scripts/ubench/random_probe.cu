// Micro-benchmark: how many random 4-byte probes per second does the H100 memory system sustain, and how many
// DRAM bytes does each one cost, for the load flavours available in PTX and for the L2 fetch-granularity limit?
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o random_probe random_probe.cu ; run: ./random_probe [GiB]
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>
typedef unsigned int u32; typedef unsigned long long u64;

template <int MODE> __device__ __forceinline__ u32 ld(const u32* p) {
    u32 v;
    if (MODE == 0) v = *p;
    else if (MODE == 1) v = __ldcg(p);
    else if (MODE == 2) v = __ldcs(p);
    else if (MODE == 3) v = __ldlu(p);
    else if (MODE == 4) v = __ldcv(p);
    else if (MODE == 5) { u64 pol; asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
                          asm volatile("ld.global.L1::no_allocate.L2::cache_hint.u32 %0, [%1], %2;" : "=r"(v) : "l"(p), "l"(pol)); }
    else { u64 pol; asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
           asm volatile("ld.global.L1::no_allocate.L2::cache_hint.u32 %0, [%1], %2;" : "=r"(v) : "l"(p), "l"(pol)); }
    return v;
}
template <int MODE, bool WRITE>
__global__ void k_probe(u32* __restrict__ tab, u64 mask, int iters, u32* out) {
    u64 x = (u64)(blockIdx.x * blockDim.x + threadIdx.x) * 0x9E3779B97F4A7C15ULL + 12345;
    u32 acc = 0;
    for (int i = 0; i < iters; i++) {
        x = x * 6364136223846793005ULL + 1442695040888963407ULL;
        u64 const idx = (x >> 20) & mask;
        u32 const v = ld<MODE>(tab + idx);
        acc += v;
        if (WRITE) tab[idx] = v + 1;
    }
    if (acc == 0x12345678) *out = acc;
}
__global__ void k_exch(u32* __restrict__ tab, u64 mask, int iters, u32* out) {      // one atomic instead of read + write
    u64 x = (u64)(blockIdx.x * blockDim.x + threadIdx.x) * 0x9E3779B97F4A7C15ULL + 12345;
    u32 acc = 0;
    for (int i = 0; i < iters; i++) {
        x = x * 6364136223846793005ULL + 1442695040888963407ULL;
        u64 const idx = (x >> 20) & mask;
        acc += atomicExch(tab + idx, (u32)i);
    }
    if (acc == 0x12345678) *out = acc;
}
__global__ void k_wonly(u32* __restrict__ tab, u64 mask, int iters, u32* out) {     // blind 4-byte writes
    u64 x = (u64)(blockIdx.x * blockDim.x + threadIdx.x) * 0x9E3779B97F4A7C15ULL + 12345;
    for (int i = 0; i < iters; i++) {
        x = x * 6364136223846793005ULL + 1442695040888963407ULL;
        tab[(x >> 20) & mask] = (u32)i;
    }
}
template <int MODE, bool WRITE> float run(u32* tab, u64 mask, int blocks, int iters, u32* out) {
    cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
    k_probe<MODE, WRITE><<<blocks, 256>>>(tab, mask, iters / 8, out);
    cudaEventRecord(a);
    k_probe<MODE, WRITE><<<blocks, 256>>>(tab, mask, iters, out);
    cudaEventRecord(b); cudaEventSynchronize(b);
    float ms = 0; cudaEventElapsedTime(&ms, a, b); return ms;
}
int main(int argc, char** argv) {
    double gib = argc > 1 ? atof(argv[1]) : 4.0;
    u64 words = 1; while (words * 4 * 2 <= (u64)(gib * (1ull << 30))) words *= 2;
    u32* tab; cudaMalloc(&tab, words * 4); cudaMemset(tab, 0, words * 4);
    u32* out; cudaMalloc(&out, 4);
    int sms = 0; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    int const blocks = sms * 8, iters = 2048;
    double const probes = (double)blocks * 256 * iters;
    {   cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b); float ms;
        k_exch<<<blocks, 256>>>(tab, words - 1, iters / 8, out); cudaEventRecord(a); k_exch<<<blocks, 256>>>(tab, words - 1, iters, out); cudaEventRecord(b); cudaEventSynchronize(b);
        cudaEventElapsedTime(&ms, a, b); printf("atomicExch (old value used)        %8.2f ms  %7.2f G probes/s\n", ms, probes / ms / 1e6);
        k_wonly<<<blocks, 256>>>(tab, words - 1, iters / 8, out); cudaEventRecord(a); k_wonly<<<blocks, 256>>>(tab, words - 1, iters, out); cudaEventRecord(b); cudaEventSynchronize(b);
        cudaEventElapsedTime(&ms, a, b); printf("blind 4-byte writes                %8.2f ms  %7.2f G probes/s\n", ms, probes / ms / 1e6); }
    const char* names[] = {"ld", "ld.cg", "ld.cs", "ld.lu", "ld.cv", "no_alloc+evict_first", "no_alloc+evict_last"};
    for (int gran : {0, 32}) {
        if (gran) { cudaError_t e = cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, gran); size_t g = 0; cudaDeviceGetLimit(&g, cudaLimitMaxL2FetchGranularity);
            printf("set L2 fetch granularity %d -> %s, now %zu\n", gran, cudaGetErrorString(e), g); }
        else { size_t g = 0; cudaDeviceGetLimit(&g, cudaLimitMaxL2FetchGranularity); printf("default L2 fetch granularity %zu\n", g); }
        float ms[7];
        ms[0] = run<0, false>(tab, words - 1, blocks, iters, out); ms[1] = run<1, false>(tab, words - 1, blocks, iters, out);
        ms[2] = run<2, false>(tab, words - 1, blocks, iters, out); ms[3] = run<3, false>(tab, words - 1, blocks, iters, out);
        ms[4] = run<4, false>(tab, words - 1, blocks, iters, out); ms[5] = run<5, false>(tab, words - 1, blocks, iters, out);
        ms[6] = run<6, false>(tab, words - 1, blocks, iters, out);
        for (int m = 0; m < 7; m++) printf("  table %.1f GiB read-only  %-22s %8.2f ms  %7.2f G probes/s\n", words * 4.0 / (1ull << 30), names[m], ms[m], probes / ms[m] / 1e6);
        float w0 = run<0, true>(tab, words - 1, blocks, iters, out), w1 = run<1, true>(tab, words - 1, blocks, iters, out);
        printf("  read+write same cell     ld    %8.2f ms  %7.2f G probes/s ; ld.cg %8.2f ms %7.2f G probes/s\n", w0, probes / w0 / 1e6, w1, probes / w1 / 1e6);
    }
    return 0;
}
