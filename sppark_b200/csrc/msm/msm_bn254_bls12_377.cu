// BN254 (alt_bn128) and BLS12-377 G1 MSM: the other two curves the reference's msm crate builds
// (poc/msm-cuda/Cargo.toml features bn254 / bls12_377, ff/alt_bn128.hpp, ff/bls12-377.hpp; the
// same pippenger.cu / pippenger_inf.cu glue with another FEATURE_*).  Reached through
// sppark_b200_msm(curve, ...) / sppark_b200_msm_dev, since one shared library serves every curve.
#include "msm_host.cuh"

RustError msm_host_bn254(void* out, const void* points, size_t npoints, const void* scalars,
                         size_t stride, bool has_flag, bool mont,
                     uint32_t scalar_bytes, uint32_t nbits)
{
    return msm_host<ff::bn254_fp_t>(out, points, npoints, scalars, stride, has_flag,
                                    mont ? scalars_from_mont<ff::bn254_fr_t> : nullptr, nullptr, nullptr,
                     scalar_bytes, nbits);
}
RustError msm_dev_bn254(void* out, const void* d_points, size_t npoints, const void* d_scalars, void* stream,
                  uint32_t scalar_bytes, uint32_t nbits)
{   return msm_dev<ff::bn254_fp_t>(out, d_points, npoints, d_scalars, stream, scalar_bytes, nbits);   }
RustError gen_points_bn254(void* d_out, size_t n, void* stream)
{   return gen_points_dev<ff::bn254_g1_gen>(d_out, n, stream);   }
RustError combine_bn254(void* out, const void* partials, size_t count)
{   return combine_host<ff::bn254_fp_t>(out, partials, count);   }

RustError msm_host_bls12_377(void* out, const void* points, size_t npoints, const void* scalars,
                             size_t stride, bool has_flag, bool mont,
                     uint32_t scalar_bytes, uint32_t nbits)
{
    return msm_host<ff::bls12_377_fp_t>(out, points, npoints, scalars, stride, has_flag,
                                        mont ? scalars_from_mont<ff::bls12_377_fr_t> : nullptr, nullptr, nullptr,
                     scalar_bytes, nbits);
}
RustError msm_dev_bls12_377(void* out, const void* d_points, size_t npoints, const void* d_scalars, void* stream,
                  uint32_t scalar_bytes, uint32_t nbits)
{   return msm_dev<ff::bls12_377_fp_t>(out, d_points, npoints, d_scalars, stream, scalar_bytes, nbits);   }
RustError gen_points_bls12_377(void* d_out, size_t n, void* stream)
{   return gen_points_dev<ff::bls12_377_g1_gen>(d_out, n, stream);   }
RustError combine_bls12_377(void* out, const void* partials, size_t count)
{   return combine_host<ff::bls12_377_fp_t>(out, partials, count);   }

RustError msm_preload_bn254(const void* points, size_t npoints, size_t stride, bool has_flag, void** d_points,
                            uint32_t* copies, uint32_t* wbits)
{   return msm_preload<ff::bn254_fp_t>(points, npoints, stride, has_flag, d_points, copies, wbits);   }
RustError msm_resident_bn254(void* out, const void* d_points, size_t npoints, const void* scalars, bool mont,
                             uint32_t wbits, uint32_t copies, size_t stride,
                       uint32_t scalar_bytes, uint32_t nbits)
{
    return msm_resident<ff::bn254_fp_t, ff::bn254_fr_t>(out, d_points, npoints, scalars, mont, wbits, copies, stride,
                   scalar_bytes, nbits);
}

RustError msm_preload_bls12_377(const void* points, size_t npoints, size_t stride, bool has_flag, void** d_points,
                                uint32_t* copies, uint32_t* wbits)
{   return msm_preload<ff::bls12_377_fp_t>(points, npoints, stride, has_flag, d_points, copies, wbits);   }
RustError msm_resident_bls12_377(void* out, const void* d_points, size_t npoints, const void* scalars, bool mont,
                                 uint32_t wbits, uint32_t copies, size_t stride,
                       uint32_t scalar_bytes, uint32_t nbits)
{
    return msm_resident<ff::bls12_377_fp_t, ff::bls12_377_fr_t>(out, d_points, npoints, scalars, mont, wbits, copies, stride,
                   scalar_bytes, nbits);
}
