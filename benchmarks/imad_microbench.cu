// Integer-pipe peak of the GPU it runs on: throughput of IMAD.WIDE.U32 (32x32+64 -> 64, the instruction the field multiply is
// made of) and of the carry-chained form IMAD.WIDE.U32.X, as a function of independent chains per thread.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o imad_microbench imad_microbench.cu ; run: ./imad_microbench
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

template <int ILP, bool CARRY>
__global__ void k(uint32_t *out, uint32_t a0, uint32_t b0, int iters) {
    uint32_t lo[ILP], hi[ILP], a[ILP];
    for (int j = 0; j < ILP; j++) { lo[j] = threadIdx.x + j; hi[j] = j; a[j] = a0 + j * 7 + threadIdx.x; }
    uint32_t b = b0 | 1;
    for (int it = 0; it < iters; it++) {
#pragma unroll
        for (int u = 0; u < 8; u++) {
#pragma unroll
            for (int j = 0; j < ILP; j++) {
                if (CARRY) asm volatile("mad.lo.cc.u32 %0, %2, %3, %0;\n\t madc.hi.cc.u32 %1, %2, %3, %1;\n\t" : "+r"(lo[j]), "+r"(hi[j]) : "r"(a[j]), "r"(b));
                else asm volatile("mad.lo.cc.u32 %0, %2, %3, %0;\n\t madc.hi.u32 %1, %2, %3, %1;\n\t" : "+r"(lo[j]), "+r"(hi[j]) : "r"(a[j]), "r"(b));
            }
        }
    }
    uint32_t s = 0;
    for (int j = 0; j < ILP; j++) s ^= lo[j] ^ hi[j];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

template <int ILP, bool CARRY>
void run(int blocks_per_sm, int threads) {
    int sms = 0, khz = 0, iters = 4096;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0); cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, 0);
    uint32_t *out; cudaMalloc(&out, (size_t)sms * blocks_per_sm * threads * 4);
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    k<ILP, CARRY><<<sms * blocks_per_sm, threads>>>(out, 3, 5, 16);
    cudaEventRecord(e0);
    k<ILP, CARRY><<<sms * blocks_per_sm, threads>>>(out, 3, 5, iters);
    cudaEventRecord(e1); cudaEventSynchronize(e1);
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    double ops = (double)sms * blocks_per_sm * threads * iters * 8.0 * ILP;      // wide multiply-adds (thread level)
    double warp_instr_per_s = ops / 32 / (ms * 1e-3);
    printf("ILP=%d carry=%d warps/SM=%d : %.1f G wide-mad/s, %.3f warp-instr/cycle/SMSP @%.3fGHz\n", ILP, (int)CARRY, blocks_per_sm * threads / 32,
           ops / (ms * 1e-3) / 1e9, warp_instr_per_s / (sms * 4.0 * khz * 1e3), khz * 1e-6);
    cudaFree(out);
}
int main() {
    cudaDeviceProp prop; cudaGetDeviceProperties(&prop, 0);
    printf("%s, %d SMs\n", prop.name, prop.multiProcessorCount);
    run<1, false>(8, 256); run<2, false>(8, 256); run<4, false>(8, 256); run<8, false>(8, 256);
    run<1, true>(8, 256); run<4, true>(8, 256); run<8, true>(8, 256);
    run<4, false>(1, 128); run<4, false>(2, 256); run<8, false>(1, 128);
    return 0;
}
