// Compute-only microbenchmark of the Goldilocks butterfly network (no memory traffic): which
// formulation of add / sub / mul issues fastest on the GPU, and what IPC a dense stream of them
// reaches.  One 16-point DFT = 32 butterflies (17 with a constant multiplication) on registers,
// the code of ntt_warp.cuh's dft_stage, repeated ITER times per thread.
//   nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -I sppark_b200/csrc -o /tmp/gl64_bfly tools/gl64_bfly_bench.cu
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
#include "ff/gl64.cuh"
#include "ntt/ntt_warp.cuh"

// ---- variants -----------------------------------------------------------------------------------
struct gl64_subc : gl64 {               // add with the add.cc -> subc idiom (5 instructions)
    static __device__ __forceinline__ T add(T a, T b)
    {
        uint32_t lo, hi, m;
        asm("{ .reg .u32 a0, a1, b0, b1;\n\t"
            "mov.b64 {a0, a1}, %3; mov.b64 {b0, b1}, %4;\n\t"
            "add.cc.u32 %0, a0, b0; addc.cc.u32 %1, a1, b1; subc.u32 %2, 0, 0;\n\t"
            "add.cc.u32 %0, %0, %2; addc.u32 %1, %1, 0; }"
            : "=r"(lo), "=r"(hi), "=r"(m) : "l"(a), "l"(b));
        return ((T)hi << 32) | lo;
    }
};
struct gl64_cmul : gl64 {               // mul written in C (mul.wide + the reduction in 64-bit C)
    static __device__ __forceinline__ T mul(T a, T b)
    {
        const uint32_t a0 = (uint32_t)a, a1 = (uint32_t)(a >> 32), b0 = (uint32_t)b, b1 = (uint32_t)(b >> 32);
        const uint64_t p00 = (uint64_t)a0 * b0, p01 = (uint64_t)a0 * b1, p10 = (uint64_t)a1 * b0, p11 = (uint64_t)a1 * b1;
        const uint64_t mid = (p00 >> 32) + (uint32_t)p01 + (uint32_t)p10;
        const uint64_t lo = (uint32_t)p00 | (mid << 32);
        const uint64_t hi = p11 + (p01 >> 32) + (p10 >> 32) + (mid >> 32);
        return mont_reduce(lo, hi);
    }
};
struct gl64_noadd : gl64 {              // NOT a field: add / sub without the wrap correction (cost floor)
    static __device__ __forceinline__ T add(T a, T b) { return a + b; }
    static __device__ __forceinline__ T sub(T a, T b) { return a - b; }
    static __device__ __forceinline__ T tight(T a) { return a; }
};
struct gl64_nomul : gl64 {              // NOT a field: the multiplication replaced by a xor (cost floor)
    static __device__ __forceinline__ T mul(T a, T b) { return a ^ b; }
};
struct gl64_notight : gl64 {            // NOT always correct: no tightening of un-multiplied operands
    static __device__ __forceinline__ T tight(T a) { return a; }
};

template<class F>
__global__ void __launch_bounds__(256, 3) bench(uint64_t* out, ntt::Tables<F> tb, int iters)
{
    typedef typename F::T T;
    T x[16];
#pragma unroll
    for (int i = 0; i < 16; i++) x[i] = (uint64_t)(threadIdx.x + 1) * 0x9E3779B97F4A7C15ull + i * 0x1234567ull + blockIdx.x;
#pragma unroll 1
    for (int it = 0; it < iters; it++) {
        ntt::dft_stage<F, 1>(x, tb);
        ntt::dft_stage<F, 2>(x, tb);
        ntt::dft_stage<F, 3>(x, tb);
        ntt::dft_stage<F, 4>(x, tb);
    }
    T acc = 0;
#pragma unroll
    for (int i = 0; i < 16; i++) acc ^= x[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = acc;
}

template<class F> void run(const char* name, int sms, double mhz)
{
    ntt::Tables<F> tb{};
    for (int i = 0; i < 8; i++) tb.w16[i] = 0x0123456789abcdefull * (i + 3) % gl64::P;
    uint64_t* out;
    cudaMalloc(&out, (size_t)sms * 3 * 256 * 8);
    const int iters = 2000;
    for (int warps_per_sm : {8, 16, 24}) {
        int blocks = sms * warps_per_sm / 8;
        bench<F><<<blocks, 256>>>(out, tb, 10);
        cudaEvent_t e0, e1;
        cudaEventCreate(&e0); cudaEventCreate(&e1);
        cudaEventRecord(e0);
        bench<F><<<blocks, 256>>>(out, tb, iters);
        cudaEventRecord(e1);
        cudaEventSynchronize(e1);
        float ms; cudaEventElapsedTime(&ms, e0, e1);
        // cycles per DFT16 (32 butterflies) per warp on one SMSP
        double dft_per_smsp = (double)warps_per_sm / 4 * iters;
        double cyc = ms * 1e-3 * mhz * 1e6 / dft_per_smsp;
        printf("%-10s warps/SM=%2d  %.3f ms  %.0f cycles per 16-point DFT per warp-slot (%.1f per butterfly)\n",
               name, warps_per_sm, ms, cyc, cyc / 32);
    }
    cudaFree(out);
}

int main()
{
    cudaDeviceProp p; cudaGetDeviceProperties(&p, 0);
    int sms = p.multiProcessorCount; double mhz = p.clockRate / 1000.0;
    printf("%s SMs=%d clock=%.0f MHz\n", p.name, sms, mhz);
    run<gl64>("current", sms, mhz);
    run<gl64_subc>("add-subc", sms, mhz);
    run<gl64_cmul>("C-mul", sms, mhz);
    run<gl64_notight>("no-tight", sms, mhz);
    run<gl64_noadd>("no-add", sms, mhz);
    run<gl64_nomul>("no-mul", sms, mhz);
    return 0;
}
