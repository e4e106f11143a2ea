// Integer-issue microbenchmark: what bounds the 384-bit Montgomery ladders?
// Measures warp-instruction throughput of IMAD.WIDE.U32 carry chains (the MSM inner loop),
// plain IMAD, and IADD3, per SM per clock.   nvcc -arch=sm_90a -O3 imad_bench.cu -o imad_bench
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

template<int MODE>
__global__ void kern(uint32_t* out, uint32_t a, uint32_t b, int iters)
{
    uint32_t x0 = threadIdx.x, x1 = a, x2 = b, x3 = a ^ b, x4 = 1, x5 = 2, x6 = 3, x7 = 4;
    for (int i = 0; i < iters; i++) {
#pragma unroll
        for (int k = 0; k < 16; k++) {
            if (MODE == 0) {           // carry-chained wide multiply-add (mad.lo.cc/madc.hi.cc pairs)
                asm volatile("mad.lo.cc.u32 %0, %4, %5, %0; madc.hi.cc.u32 %1, %4, %5, %1;"
                             "madc.lo.cc.u32 %2, %4, %6, %2; madc.hi.u32 %3, %4, %6, %3;"
                             : "+r"(x0), "+r"(x1), "+r"(x2), "+r"(x3) : "r"(a), "r"(b), "r"(x4));
                asm volatile("mad.lo.cc.u32 %0, %4, %5, %0; madc.hi.cc.u32 %1, %4, %5, %1;"
                             "madc.lo.cc.u32 %2, %4, %6, %2; madc.hi.u32 %3, %4, %6, %3;"
                             : "+r"(x4), "+r"(x5), "+r"(x6), "+r"(x7) : "r"(a), "r"(b), "r"(x0));
            } else if (MODE == 1) {    // independent 32-bit IMAD
                x0 = x0 * a + b; x1 = x1 * a + b; x2 = x2 * a + b; x3 = x3 * a + b;
                x4 = x4 * a + b; x5 = x5 * a + b; x6 = x6 * a + b; x7 = x7 * a + b;
            } else if (MODE == 2) {    // independent adds (alu pipe)
                asm volatile("add.u32 %0, %0, %1;" : "+r"(x0) : "r"(a));
                asm volatile("add.u32 %0, %0, %1;" : "+r"(x1) : "r"(a));
                asm volatile("add.u32 %0, %0, %1;" : "+r"(x2) : "r"(a));
                asm volatile("add.u32 %0, %0, %1;" : "+r"(x3) : "r"(a));
                asm volatile("add.u32 %0, %0, %1;" : "+r"(x4) : "r"(a));
                asm volatile("add.u32 %0, %0, %1;" : "+r"(x5) : "r"(a));
                asm volatile("add.u32 %0, %0, %1;" : "+r"(x6) : "r"(a));
                asm volatile("add.u32 %0, %0, %1;" : "+r"(x7) : "r"(a));
            } else {                   // mixed: 4 wide mads + 4 adds
                asm volatile("mad.lo.cc.u32 %0, %4, %5, %0; madc.hi.cc.u32 %1, %4, %5, %1;"
                             "madc.lo.cc.u32 %2, %4, %6, %2; madc.hi.u32 %3, %4, %6, %3;"
                             : "+r"(x0), "+r"(x1), "+r"(x2), "+r"(x3) : "r"(a), "r"(b), "r"(x4));
                asm volatile("add.u32 %0, %0, %1;" : "+r"(x4) : "r"(a));
                asm volatile("add.u32 %0, %0, %1;" : "+r"(x5) : "r"(a));
                asm volatile("add.u32 %0, %0, %1;" : "+r"(x6) : "r"(a));
                asm volatile("add.u32 %0, %0, %1;" : "+r"(x7) : "r"(a));
            }
        }
    }
    out[blockIdx.x * blockDim.x + threadIdx.x] = x0 ^ x1 ^ x2 ^ x3 ^ x4 ^ x5 ^ x6 ^ x7;
}

template<int MODE> void run(const char* name, int instr_per_iter, int sms, double mhz)
{
    uint32_t* out;
    cudaMalloc(&out, sms * 8 * 1024 * 4);
    for (int warps = 4; warps <= 32; warps *= 2) {
        int threads = warps * 32 > 1024 ? 1024 : warps * 32;
        int blocks = sms * (warps * 32 / threads);
        cudaEvent_t e0, e1;
        cudaEventCreate(&e0); cudaEventCreate(&e1);
        int iters = 4096;
        kern<MODE><<<blocks, threads>>>(out, 3, 5, 16);
        cudaEventRecord(e0);
        kern<MODE><<<blocks, threads>>>(out, 3, 5, iters);
        cudaEventRecord(e1);
        cudaEventSynchronize(e1);
        float ms; cudaEventElapsedTime(&ms, e0, e1);
        double winstr = (double)blocks * (threads / 32) * iters * 16.0 * instr_per_iter;
        double per_sm_clk = winstr / (ms * 1e-3) / sms / (mhz * 1e6);
        printf("%-28s warps/SM=%2d  %.3f ms  %.2f warp-instr/clk/SM (at %.0f MHz nominal)  %.1f G thread-instr/s\n",
               name, warps, ms, per_sm_clk, mhz, winstr * 32 / (ms * 1e-3) / 1e9);
    }
    cudaFree(out);
}

int main()
{
    cudaDeviceProp p; cudaGetDeviceProperties(&p, 0);
    int sms = p.multiProcessorCount; double mhz = p.clockRate / 1000.0;
    printf("%s SMs=%d clock=%.0f MHz\n", p.name, sms, mhz);
    run<0>("mad.wide carry chain (4/asm)", 8, sms, mhz);   // PTX-level count; SASS fuses lo/hi pairs -> 4 IMAD.WIDE
    run<1>("IMAD 32-bit independent", 8, sms, mhz);
    run<2>("IADD independent", 8, sms, mhz);
    run<3>("mixed 2 wide + 4 add (PTX 8)", 8, sms, mhz);
    return 0;
}
