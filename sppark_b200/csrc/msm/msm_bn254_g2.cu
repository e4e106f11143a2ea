// BN254 G2 MSM: mult_pippenger_fp2_inf of the reference's bn254 build
// (poc/msm-cuda/cuda/pippenger_inf.cu:8-13,36-47 with FEATURE_BN254; ff/alt_bn128-fp2.hpp: Fp2 = Fp[u]/(u^2 + 1)).
// Same sort / accumulate / reduce kernels as G1, instantiated over ff::fp2_t (ff/fp2.cuh).  Reached
// through sppark_b200_msm(SPPARK_CURVE_BN254_G2, ...): one shared library serves every curve,
// the symbol mult_pippenger_fp2_inf itself is the BLS12-381 one (msm_bls12_381_g2.cu).
#include "msm_host.cuh"
#include "../ff/fp2.cuh"

namespace {
typedef ff::fp2_t<ff::bn254_fp_t, 1> fp2;
struct g2_gen : ff::bn254_g2_gen { typedef fp2 F; };
}

RustError msm_host_bn254_g2(void* out, const void* points, size_t npoints, const void* scalars,
                              size_t stride, bool has_flag, bool mont,
                     uint32_t scalar_bytes, uint32_t nbits)
{
    return msm_host<fp2>(out, points, npoints, scalars, stride, has_flag,
                         mont ? scalars_from_mont<ff::bn254_fr_t> : nullptr, nullptr, nullptr,
                     scalar_bytes, nbits);
}
RustError msm_dev_bn254_g2(void* out, const void* d_points, size_t npoints, const void* d_scalars, void* stream,
                  uint32_t scalar_bytes, uint32_t nbits)
{   return msm_dev<fp2>(out, d_points, npoints, d_scalars, stream, scalar_bytes, nbits);   }
RustError gen_points_bn254_g2(void* d_out, size_t n, void* stream)
{   return gen_points_dev<g2_gen>(d_out, n, stream);   }
RustError combine_bn254_g2(void* out, const void* partials, size_t count)
{   return combine_host<fp2>(out, partials, count);   }
RustError msm_preload_bn254_g2(const void* points, size_t npoints, size_t stride, bool has_flag, void** d_points,
                               uint32_t* copies, uint32_t* wbits)
{   return msm_preload<fp2>(points, npoints, stride, has_flag, d_points, copies, wbits);   }
RustError msm_resident_bn254_g2(void* out, const void* d_points, size_t npoints, const void* scalars, bool mont,
                                uint32_t wbits, uint32_t copies, size_t stride,
                       uint32_t scalar_bytes, uint32_t nbits)
{
    return msm_resident<fp2, ff::bn254_fr_t>(out, d_points, npoints, scalars, mont, wbits, copies, stride,
                   scalar_bytes, nbits);
}
