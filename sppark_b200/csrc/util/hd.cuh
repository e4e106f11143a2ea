// Host/device portability macros.  Every arithmetic and index-mapping routine of the
// hot path is written HD so that tests/emu/*.cpp can single-step the exact kernel logic
// on the CPU (phase by phase) before it is run on the GPU.  The product path itself is
// CUDA only: nothing here provides a CPU fallback for the C-ABI entry points.
#pragma once
#include <cstddef>
#include <cstdint>
#if defined(__CUDACC__)
# define HD __host__ __device__ __forceinline__
# define DEV __device__ __forceinline__
# define HD_NOINLINE __host__ __device__ __noinline__
#else
# define HD inline
# define DEV inline
# define HD_NOINLINE
#endif

HD uint32_t brev32(uint32_t x, uint32_t nbits)
{
    if (nbits == 0) return 0;
#if defined(__CUDA_ARCH__)
    return __brev(x) >> (32 - nbits);
#else
    x = ((x >> 1) & 0x55555555u) | ((x & 0x55555555u) << 1);
    x = ((x >> 2) & 0x33333333u) | ((x & 0x33333333u) << 2);
    x = ((x >> 4) & 0x0f0f0f0fu) | ((x & 0x0f0f0f0fu) << 4);
    x = ((x >> 8) & 0x00ff00ffu) | ((x & 0x00ff00ffu) << 8);
    x = (x >> 16) | (x << 16);
    return x >> (32 - nbits);
#endif
}
