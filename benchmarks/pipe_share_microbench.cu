// Do DFMA (FP64) and IMAD.WIDE.U32 (the wide integer multiply-add the field arithmetic is made of) run on separate pipes on this GPU?
// Four kernels at full occupancy, the same work per thread in each class:
//   I : 8 independent IMAD.WIDE chains            D : 8 independent DFMA chains
//   M : both, interleaved in one instruction stream (every thread issues the I work and the D work)
//   W : warp-specialised -- even warps run the I loop, odd warps the D loop, each with the doubled trip count (same total work as M)
// Separate pipes: t(M) ~ t(W) ~ max(t(I), t(D)).   One shared unit: t(M) ~ t(W) ~ t(I) + t(D).
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o pipe_share_microbench pipe_share_microbench.cu ; run: ./pipe_share_microbench
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

#define NCH 8
__device__ __forceinline__ void imad_step(uint32_t (&lo)[NCH], uint32_t (&hi)[NCH], const uint32_t (&a)[NCH], uint32_t b) {
#pragma unroll
    for (int j = 0; j < NCH; j++) asm volatile("mad.lo.cc.u32 %0, %2, %3, %0;\n\t madc.hi.u32 %1, %2, %3, %1;\n\t" : "+r"(lo[j]), "+r"(hi[j]) : "r"(a[j]), "r"(b));
}
__device__ __forceinline__ void dfma_step(double (&x)[NCH], double m, double c) {
#pragma unroll
    for (int j = 0; j < NCH; j++) asm volatile("fma.rz.f64 %0, %0, %1, %2;" : "+d"(x[j]) : "d"(m), "d"(c));
}
// mode 0 = I, 1 = D, 2 = M, 3 = W
template <int MODE>
__global__ void __launch_bounds__(256) k(uint32_t *out, uint32_t a0, uint32_t b0, double m, double c, int iters) {
    uint32_t lo[NCH], hi[NCH], a[NCH]; double x[NCH];
    for (int j = 0; j < NCH; j++) { lo[j] = threadIdx.x + j; hi[j] = j; a[j] = a0 + j * 7 + threadIdx.x; x[j] = 1.0 + 1e-3 * (threadIdx.x + j); }
    const uint32_t b = b0 | 1;
    const bool odd_warp = (threadIdx.x >> 5) & 1;
    for (int it = 0; it < iters; it++) {
#pragma unroll
        for (int u = 0; u < 8; u++) {
            if (MODE == 0) imad_step(lo, hi, a, b);
            else if (MODE == 1) dfma_step(x, m, c);
            else if (MODE == 2) { imad_step(lo, hi, a, b); dfma_step(x, m, c); }
            else { if (odd_warp) { dfma_step(x, m, c); dfma_step(x, m, c); } else { imad_step(lo, hi, a, b); imad_step(lo, hi, a, b); } }
        }
    }
    uint32_t s = 0;
    for (int j = 0; j < NCH; j++) s ^= lo[j] ^ hi[j] ^ (uint32_t)__double_as_longlong(x[j]);
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
template <int MODE> float run(uint32_t *out, int blocks, int iters) {
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    k<MODE><<<blocks, 256>>>(out, 3, 5, 1.0000001, 1e-9, 16);
    float best = 1e30f;
    for (int rep = 0; rep < 3; rep++) {
        cudaEventRecord(e0); k<MODE><<<blocks, 256>>>(out, 3, 5, 1.0000001, 1e-9, iters); cudaEventRecord(e1); cudaEventSynchronize(e1);
        float ms; cudaEventElapsedTime(&ms, e0, e1); if (ms < best) best = ms;
    }
    return best;
}
int main() {
    int sms = 0; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    const int per_sm = 8, blocks = sms * per_sm, iters = 2048;       // 64 warps per SM
    uint32_t *out; cudaMalloc(&out, (size_t)blocks * 256 * 4);
    float tI = run<0>(out, blocks, iters), tD = run<1>(out, blocks, iters), tM = run<2>(out, blocks, iters), tW = run<3>(out, blocks, iters);
    double n = (double)blocks * 256 * iters * 8.0 * NCH;             // instructions of one class, thread level
    printf("{\"sms\": %d, \"warps_per_sm\": %d, \"imad_wide_ms\": %.3f, \"dfma_ms\": %.3f, \"interleaved_ms\": %.3f, \"warp_specialised_ms\": %.3f, "
           "\"imad_wide_T_per_s\": %.2f, \"dfma_T_per_s\": %.2f, \"interleaved_over_sum\": %.3f, \"interleaved_over_max\": %.3f, \"warp_specialised_over_sum\": %.3f, \"warp_specialised_over_max\": %.3f}\n",
           sms, per_sm * 8, tI, tD, tM, tW, n / (tI * 1e-3) / 1e12, n / (tD * 1e-3) / 1e12, tM / (tI + tD), tM / (tI > tD ? tI : tD), tW / (tI + tD), tW / (tI > tD ? tI : tD));
    cudaFree(out);
    return 0;
}
