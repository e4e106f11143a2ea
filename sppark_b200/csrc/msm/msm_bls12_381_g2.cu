// BLS12-381 G2 MSM: the curve of the third entry point of poc/msm-cuda's default (bls12_381) build,
//   mult_pippenger_fp2_inf   poc/msm-cuda/cuda/pippenger_inf.cu:36-43 (defined in msm.cu)
// Same sort / accumulate / reduce kernels as G1, instantiated over Fp2 (ff/fp2.cuh).
#include "msm_host.cuh"
#include "../ff/fp2.cuh"

namespace {
typedef ff::fp2_t<ff::bls12_381_fp_t> fp2;
struct g2_gen : ff::bls12_381_g2_gen { typedef fp2 F; };
}

constexpr curve_ops curve_bls12_381_g2 = curve_row<g2_gen, ff::bls12_381_fr_t>();
