// BLS12-381 G2 MSM: the third entry point of poc/msm-cuda's default (bls12_381) build,
//   mult_pippenger_fp2_inf   poc/msm-cuda/cuda/pippenger_inf.cu:36-43
// Same sort / accumulate / reduce kernels as G1, instantiated over Fp2 (ff/fp2.cuh).
#include "msm_host.cuh"
#include "../ff/fp2.cuh"

namespace {
typedef ff::fp2_t<ff::bls12_381_fp_t> fp2;
struct g2_gen : ff::bls12_381_g2_gen { typedef fp2 F; };
}

RustError msm_host_bls12_381_g2(void* out, const void* points, size_t npoints, const void* scalars,
                                size_t stride, bool has_flag, bool mont,
                     uint32_t scalar_bytes, uint32_t nbits)
{
    return msm_host<fp2>(out, points, npoints, scalars, stride, has_flag,
                         mont ? scalars_from_mont<ff::bls12_381_fr_t> : nullptr, nullptr, nullptr,
                     scalar_bytes, nbits);
}
RustError msm_dev_bls12_381_g2(void* out, const void* d_points, size_t npoints, const void* d_scalars, void* stream,
                  uint32_t scalar_bytes, uint32_t nbits)
{   return msm_dev<fp2>(out, d_points, npoints, d_scalars, stream, scalar_bytes, nbits);   }
RustError gen_points_bls12_381_g2(void* d_out, size_t n, void* stream)
{   return gen_points_dev<g2_gen>(d_out, n, stream);   }
RustError combine_bls12_381_g2(void* out, const void* partials, size_t count)
{   return combine_host<fp2>(out, partials, count);   }

extern "C" RustError mult_pippenger_fp2_inf(void* out, const void* points, size_t npoints,
                                            const void* scalars, size_t ffi_affine_sz)
{   return msm_host_bls12_381_g2(out, points, npoints, scalars, ffi_affine_sz, true, false, 32, 255);   }

RustError msm_preload_bls12_381_g2(const void* points, size_t npoints, size_t stride, bool has_flag, void** d_points,
                                   uint32_t* copies, uint32_t* wbits)
{   return msm_preload<fp2>(points, npoints, stride, has_flag, d_points, copies, wbits);   }
RustError msm_resident_bls12_381_g2(void* out, const void* d_points, size_t npoints, const void* scalars, bool mont,
                                    uint32_t wbits, uint32_t copies, size_t stride,
                       uint32_t scalar_bytes, uint32_t nbits)
{
    return msm_resident<fp2, ff::bls12_381_fr_t>(out, d_points, npoints, scalars, mont, wbits, copies, stride,
                   scalar_bytes, nbits);
}
