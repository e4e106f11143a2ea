// Pallas / Vesta MSM (BASELINE.json config 4; the reference has no PoC boundary for Pasta, so
// these are reached through sppark_b200_msm / sppark_b200_msm_dev).
#include "msm_host.cuh"

// scalar fields: Pallas' group order is Vesta's base-field modulus and vice versa (ff/pasta.hpp:92-103)
RustError msm_host_pallas(void* out, const void* points, size_t npoints, const void* scalars,
                          size_t stride, bool has_flag, bool mont,
                     uint32_t scalar_bytes, uint32_t nbits)
{
    return msm_host<ff::pallas_fp_t>(out, points, npoints, scalars, stride, has_flag,
                                     mont ? scalars_from_mont<ff::vesta_fp_t> : nullptr, nullptr, nullptr,
                     scalar_bytes, nbits);
}
RustError msm_dev_pallas(void* out, const void* d_points, size_t npoints, const void* d_scalars, void* stream,
                  uint32_t scalar_bytes, uint32_t nbits)
{   return msm_dev<ff::pallas_fp_t>(out, d_points, npoints, d_scalars, stream, scalar_bytes, nbits);   }
RustError msm_host_vesta(void* out, const void* points, size_t npoints, const void* scalars,
                         size_t stride, bool has_flag, bool mont,
                     uint32_t scalar_bytes, uint32_t nbits)
{
    return msm_host<ff::vesta_fp_t>(out, points, npoints, scalars, stride, has_flag,
                                    mont ? scalars_from_mont<ff::pallas_fp_t> : nullptr, nullptr, nullptr,
                     scalar_bytes, nbits);
}
RustError msm_dev_vesta(void* out, const void* d_points, size_t npoints, const void* d_scalars, void* stream,
                  uint32_t scalar_bytes, uint32_t nbits)
{   return msm_dev<ff::vesta_fp_t>(out, d_points, npoints, d_scalars, stream, scalar_bytes, nbits);   }
RustError gen_points_pallas(void* d_out, size_t n, void* stream)
{   return gen_points_dev<ff::pallas_gen>(d_out, n, stream);   }
RustError gen_points_vesta(void* d_out, size_t n, void* stream)
{   return gen_points_dev<ff::vesta_gen>(d_out, n, stream);   }
RustError combine_pallas(void* out, const void* partials, size_t count)
{   return combine_host<ff::pallas_fp_t>(out, partials, count);   }
RustError combine_vesta(void* out, const void* partials, size_t count)
{   return combine_host<ff::vesta_fp_t>(out, partials, count);   }

RustError msm_preload_pallas(const void* points, size_t npoints, size_t stride, bool has_flag, void** d_points,
                             uint32_t* copies, uint32_t* wbits)
{   return msm_preload<ff::pallas_fp_t>(points, npoints, stride, has_flag, d_points, copies, wbits);   }
RustError msm_resident_pallas(void* out, const void* d_points, size_t npoints, const void* scalars, bool mont,
                              uint32_t wbits, uint32_t copies, size_t stride,
                       uint32_t scalar_bytes, uint32_t nbits)
{
    return msm_resident<ff::pallas_fp_t, ff::vesta_fp_t>(out, d_points, npoints, scalars, mont, wbits, copies, stride,
                   scalar_bytes, nbits);
}

RustError msm_preload_vesta(const void* points, size_t npoints, size_t stride, bool has_flag, void** d_points,
                            uint32_t* copies, uint32_t* wbits)
{   return msm_preload<ff::vesta_fp_t>(points, npoints, stride, has_flag, d_points, copies, wbits);   }
RustError msm_resident_vesta(void* out, const void* d_points, size_t npoints, const void* scalars, bool mont,
                             uint32_t wbits, uint32_t copies, size_t stride,
                       uint32_t scalar_bytes, uint32_t nbits)
{
    return msm_resident<ff::vesta_fp_t, ff::pallas_fp_t>(out, d_points, npoints, scalars, mont, wbits, copies, stride,
                   scalar_bytes, nbits);
}
