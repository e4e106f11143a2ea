// One dispatch row per MSM curve: the entry points its curve file instantiates from the templates
// of msm_host.cuh (curve_row) and its packed layouts.  Each row is defined constexpr in its curve
// file (msm_bls12_381.cu, msm_pasta.cu, msm_bn254_bls12_377.cu, msm_*_g2.cu), so it is constant-
// initialized: no other unit depends on the order in which static initializers run.
// The functions take checked arguments (msm.cu) and throw on failure.
#pragma once
#include "../../../include/sppark_b200.h"

// host affine rows of `stride` bytes, an infinity byte after Y when has_flag
struct host_rows {
    const void* p;
    size_t stride;
    bool has_flag;
};

// the points of a host-scalar MSM: host rows, or (d_rows set) a context's device rows -- packed rows, or
// with copies > 1 a precomputed table of width wbits whose copies lie copy_stride rows apart
struct msm_points {
    host_rows host;
    const void* d_rows;
    uint32_t wbits, copies;
    size_t copy_stride;
};

// mont: scalars in Montgomery form; scalar_bytes, nbits: the scalar format (32, 255 for 32-byte
// scalars); batch: vectors of npoints scalars one after the other, one Jacobian point per vector
struct curve_ops {
    void (*msm)(void* out, const msm_points& points, size_t npoints, const void* scalars, size_t batch, bool mont,
                uint32_t scalar_bytes, uint32_t nbits);
    void (*dev)(void* out, const void* d_points, size_t npoints, const void* d_scalars, size_t batch, void* stream,
                uint32_t scalar_bytes, uint32_t nbits);
    void (*preload)(const host_rows& rows, size_t npoints, void** d_points, uint32_t* copies, uint32_t* wbits);
    // out[i] = s_i * P_i as packed affine rows (msm_scale.cuh), from host rows or device rows
    void (*scale)(void* out, const host_rows& rows, size_t npoints, const void* scalars, uint32_t scalar_bytes,
                  uint32_t nbits);
    void (*scale_dev)(void* d_out, const void* d_points, size_t npoints, const void* d_scalars, uint32_t scalar_bytes,
                      uint32_t nbits, void* stream);
    void (*gen)(void* d_out, size_t n, void* stream);
    void (*combine)(void* out, const void* partials, size_t count);
    size_t affine_bytes, jacobian_bytes;        // packed {X, Y} and {X, Y, Z}
};

// hidden: the rows join the library's own units and are not part of its ABI; they stay out of its
// exported symbols, so no other definition of these names can take their place at load time
__attribute__((visibility("hidden"))) extern const curve_ops curve_bls12_381, curve_pallas, curve_vesta,
    curve_bls12_381_g2, curve_bn254, curve_bls12_377, curve_bn254_g2, curve_bls12_377_g2;
