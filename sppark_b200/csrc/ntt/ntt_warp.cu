// Warp-autonomous NTT passes (ntt_warp.cuh) for the single-word fields: instantiations and launcher.
#include "../ff/field_dispatch.cuh"
#include "ntt_plan.hpp"
#include "ntt_warp.cuh"

namespace ntt {
// ---- warp-autonomous passes (ntt_warp.cuh) ---------------------------------------------------
template<class F, uint32_t R, uint32_t CPT, uint32_t TW>
static void launch_warp_tw(const gpu_t& gpu, const Pass& d, const Tables<F>& tb, const typename F::T* in,
                              typename F::T* out, uint32_t ncols, cudaStream_t stream)
{
    constexpr uint32_t WARPS = 8, SPW = 32u >> (R - 4);
    const size_t smem = (size_t)cta_smem_words(R, CPT, WARPS) * sizeof(typename F::T);
    // per device (function attributes and occupancy are per context): resident CTAs per SM
    static int per_sm[64];
    int& ctas = per_sm[gpu.cid() & 63];
    if (ctas == 0) {
        CUDA_OK(cudaFuncSetAttribute(pass_kernel_warp<F, R, CPT, TW>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctas, pass_kernel_warp<F, R, CPT, TW>, WARPS * 32, smem));
        if (ctas < 1) throw cuda_error(-(int)cudaErrorLaunchOutOfResources, "NTT warp pass does not fit an SM");
    }
    // persistent warps: at most one resident wave, every warp walks units with the grid's stride
    const uint32_t units = (ncols + SPW * CPT - 1) / (SPW * CPT);
    uint32_t grid = (units + WARPS - 1) / WARPS;
    const uint32_t wave = (uint32_t)gpu.sm_count() * (uint32_t)ctas;
    if (grid > wave) grid = wave;
    pass_kernel_warp<F, R, CPT, TW><<<grid, WARPS * 32, smem, stream>>>(d, tb, in, out, ncols);
}

template<class F, uint32_t R, uint32_t CPT>
static void launch_warp_shape(const gpu_t& gpu, const Pass& d, const Tables<F>& tb, const typename F::T* in,
                              typename F::T* out, uint32_t ncols, cudaStream_t stream)
{
    switch (d.tw_mode) {
    case TW_LOAD: launch_warp_tw<F, R, CPT, TW_LOAD>(gpu, d, tb, in, out, ncols, stream); break;
    case TW_STORE: launch_warp_tw<F, R, CPT, TW_STORE>(gpu, d, tb, in, out, ncols, stream); break;
    default: launch_warp_tw<F, R, CPT, TW_NONE>(gpu, d, tb, in, out, ncols, stream); break;
    }
}

template<class F, uint32_t CPT>
static bool launch_warp_cpt(const gpu_t& gpu, const Pass& d, const Tables<F>& tb, const typename F::T* in,
                            typename F::T* out, uint32_t ncols, cudaStream_t stream)
{
    switch (d.lg_r) {
    case 4: launch_warp_shape<F, 4, CPT>(gpu, d, tb, in, out, ncols, stream); return true;
    case 5: launch_warp_shape<F, 5, CPT>(gpu, d, tb, in, out, ncols, stream); return true;
    case 6: launch_warp_shape<F, 6, CPT>(gpu, d, tb, in, out, ncols, stream); return true;
    case 7: launch_warp_shape<F, 7, CPT>(gpu, d, tb, in, out, ncols, stream); return true;
    case 8: launch_warp_shape<F, 8, CPT>(gpu, d, tb, in, out, ncols, stream); return true;
    default: return false;
    }
}

template<class F> bool launch_warp(const gpu_t& gpu, const Pass& d, const Tables<F>& tb, const typename F::T* in,
                                   typename F::T* out, uint32_t ncols, cudaStream_t stream)
{
    // columns per lane: 1 for 8-byte words, 2 for 4-byte words (a warp then always moves at
    // least 16 bytes per row); SPPARK_B200_NTT_CPT overrides (experiments)
    uint32_t cpt = sizeof(typename F::T) == 4 ? 2 : 1;
    if (const char* env = getenv("SPPARK_B200_NTT_CPT")) cpt = (uint32_t)atoi(env);
    return cpt == 2 ? launch_warp_cpt<F, 2>(gpu, d, tb, in, out, ncols, stream)
                    : launch_warp_cpt<F, 1>(gpu, d, tb, in, out, ncols, stream);
}
template bool launch_warp<gl64>(const gpu_t&, const Pass&, const Tables<gl64>&, const uint64_t*, uint64_t*, uint32_t, cudaStream_t);
template bool launch_warp<bb31>(const gpu_t&, const Pass&, const Tables<bb31>&, const uint32_t*, uint32_t*, uint32_t, cudaStream_t);


// ---- known-answer hook: the device field arithmetic of the single-word fields ------------------
// op 0: mul (second operand a canonical Montgomery-form constant), 1: add, 2: sub (second operand
// canonical), 3: tight, 4: canon; op 100 (gl64, experiments): add with the add.cc -> subc idiom
__device__ __forceinline__ uint64_t gl64_add_subc(uint64_t a, uint64_t b)
{
    uint32_t lo, hi, m;
    asm("{ .reg .u32 a0, a1, b0, b1;\n\t"
        "mov.b64 {a0, a1}, %3; mov.b64 {b0, b1}, %4;\n\t"
        "add.cc.u32 %0, a0, b0; addc.cc.u32 %1, a1, b1; subc.u32 %2, 0, 0;\n\t"
        "add.cc.u32 %0, %0, %2; addc.u32 %1, %1, 0; }"
        : "=r"(lo), "=r"(hi), "=r"(m) : "l"(a), "l"(b));
    return ((uint64_t)hi << 32) | lo;
}
template<class F>
__global__ void word_selftest_kernel(int op, size_t n, typename F::T* r, const typename F::T* a, const typename F::T* b)
{
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const typename F::T x = a[i], y = b[i];
    typename F::T z;
    switch (op) {
    case 0: z = F::mul(x, y); break;
    case 1: z = F::add(x, y); break;
    case 2: z = F::sub(x, y); break;
    case 3: z = F::tight(x); break;
    case 100:
        if constexpr (sizeof(typename F::T) == 8) z = gl64_add_subc(x, y);
        else z = F::add(x, y);
        break;
    default: z = F::canon(x); break;
    }
    r[i] = z;
}

}  // namespace ntt

extern "C" RustError sppark_b200_selftest_word_field(int field, int op, size_t n, void* r, const void* a, const void* b)
{
    return with_word_field(field, "selftest_word_field: unknown field", nullptr, [&](auto t) {
        typedef typename decltype(t)::type F;
        typedef typename F::T T;
        return guarded([&] {
            const gpu_t& gpu = select_gpu(-1);
            const stream_t& s = gpu[0];
            dev_ptr_t<T> da(n, s), db(n, s), dr(n, s);
            s.HtoD(da, a, n * sizeof(T));
            s.HtoD(db, b, n * sizeof(T));
            ntt::word_selftest_kernel<F><<<(unsigned)((n + 127) / 128), 128, 0, s>>>(op, n, dr, da, db);
            COUNT_LAUNCH();
            CUDA_OK(cudaGetLastError());
            s.DtoH(r, dr, n * sizeof(T));
            s.sync();
            return rust_ok();
        });
    });
}
