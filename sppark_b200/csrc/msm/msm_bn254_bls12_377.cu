// BN254 (alt_bn128) and BLS12-377 G1 MSM: the other two curves the reference's msm crate builds
// (poc/msm-cuda/Cargo.toml features bn254 / bls12_377, ff/alt_bn128.hpp, ff/bls12-377.hpp; the
// same pippenger.cu / pippenger_inf.cu glue with another FEATURE_*).  Reached through
// sppark_b200_msm(curve, ...) / sppark_b200_msm_dev, since one shared library serves every curve.
#include "msm_host.cuh"

constexpr curve_ops curve_bn254 = curve_row<ff::bn254_g1_gen, ff::bn254_fr_t>();
constexpr curve_ops curve_bls12_377 = curve_row<ff::bls12_377_g1_gen, ff::bls12_377_fr_t>();
