// BLS12-377 G2 MSM: mult_pippenger_fp2_inf of the reference's bls12_377 build
// (poc/msm-cuda/cuda/pippenger_inf.cu:8-13,36-47 with FEATURE_BLS12_377; ff/bls12-377-fp2.hpp: Fp2 = Fp[u]/(u^2 + 5)).
// Same sort / accumulate / reduce kernels as G1, instantiated over ff::fp2_t (ff/fp2.cuh).  Reached
// through sppark_b200_msm(SPPARK_CURVE_BLS12_377_G2, ...): one shared library serves every curve,
// the symbol mult_pippenger_fp2_inf itself is the BLS12-381 one (msm.cu).
#include "msm_host.cuh"
#include "../ff/fp2.cuh"

namespace {
typedef ff::fp2_t<ff::bls12_377_fp_t, 5> fp2;
struct g2_gen : ff::bls12_377_g2_gen { typedef fp2 F; };
}

constexpr curve_ops curve_bls12_377_g2 = curve_row<g2_gen, ff::bls12_377_fr_t>();
