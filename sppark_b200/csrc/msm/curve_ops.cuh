// One dispatch row per MSM curve: the entry points its curve file instantiates from the templates
// of msm_host.cuh (curve_row) and its packed layouts.  Each row is defined constexpr in its curve
// file (msm_bls12_381.cu, msm_pasta.cu, msm_bn254_bls12_377.cu, msm_*_g2.cu), so it is constant-
// initialized: no other unit depends on the order in which static initializers run.
#pragma once
#include "../../../include/sppark_b200.h"

// stride: bytes per host affine row; has_flag: an infinity byte follows Y; mont: scalars in
// Montgomery form; scalar_bytes, nbits: the scalar format (32, 255 for 32-byte scalars)
struct curve_ops {
    RustError (*host)(void* out, const void* points, size_t npoints, const void* scalars, size_t stride,
                      bool has_flag, bool mont, uint32_t scalar_bytes, uint32_t nbits);
    RustError (*dev)(void* out, const void* d_points, size_t npoints, const void* d_scalars, void* stream,
                     uint32_t scalar_bytes, uint32_t nbits);
    RustError (*gen)(void* d_out, size_t n, void* stream);
    RustError (*combine)(void* out, const void* partials, size_t count);
    RustError (*preload)(const void* points, size_t npoints, size_t stride, bool has_flag, void** d_points,
                         uint32_t* copies, uint32_t* wbits);
    RustError (*resident)(void* out, const void* d_points, size_t npoints, const void* scalars, bool mont,
                          uint32_t wbits, uint32_t copies, size_t copy_stride, uint32_t scalar_bytes, uint32_t nbits);
    // batches: `batch` vectors of npoints scalars one after the other, one Jacobian point per vector
    RustError (*resident_batch)(void* out, const void* d_points, size_t npoints, const void* scalars, size_t batch,
                                bool mont, uint32_t wbits, uint32_t copies, size_t copy_stride, uint32_t scalar_bytes,
                                uint32_t nbits);
    RustError (*dev_batch)(void* out, const void* d_points, size_t npoints, const void* d_scalars, size_t batch,
                           void* stream, uint32_t scalar_bytes, uint32_t nbits);
    // out[i] = s_i * P_i as packed affine rows (msm_scale.cuh): host rows at `stride` bytes, or device rows
    RustError (*scale)(void* out, const void* points, size_t npoints, const void* scalars, size_t stride,
                       bool has_flag, uint32_t scalar_bytes, uint32_t nbits);
    RustError (*scale_dev)(void* d_out, const void* d_points, size_t npoints, const void* d_scalars,
                           uint32_t scalar_bytes, uint32_t nbits, void* stream);
    size_t affine_bytes, jacobian_bytes;        // packed {X, Y} and {X, Y, Z}
};

// hidden: the rows join the library's own units and are not part of its ABI; they stay out of its
// exported symbols, so no other definition of these names can take their place at load time
__attribute__((visibility("hidden"))) extern const curve_ops curve_bls12_381, curve_pallas, curve_vesta,
    curve_bls12_381_g2, curve_bn254, curve_bls12_377, curve_bn254_g2, curve_bls12_377_g2;
