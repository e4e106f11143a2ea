// BN254 G2 MSM: mult_pippenger_fp2_inf of the reference's bn254 build
// (poc/msm-cuda/cuda/pippenger_inf.cu:8-13,36-47 with FEATURE_BN254; ff/alt_bn128-fp2.hpp: Fp2 = Fp[u]/(u^2 + 1)).
// Same sort / accumulate / reduce kernels as G1, instantiated over ff::fp2_t (ff/fp2.cuh).  Reached
// through sppark_b200_msm(SPPARK_CURVE_BN254_G2, ...): one shared library serves every curve,
// the symbol mult_pippenger_fp2_inf itself is the BLS12-381 one (msm.cu).
#include "msm_host.cuh"
#include "../ff/fp2.cuh"

namespace {
typedef ff::fp2_t<ff::bn254_fp_t, 1> fp2;
struct g2_gen : ff::bn254_g2_gen { typedef fp2 F; };
}

constexpr curve_ops curve_bn254_g2 = curve_row<g2_gen, ff::bn254_fr_t>();
