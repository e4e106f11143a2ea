// Pallas / Vesta MSM (BASELINE.json config 4; the reference has no PoC boundary for Pasta, so
// these are reached through sppark_b200_msm / sppark_b200_msm_dev).
#include "msm_host.cuh"

// scalar fields: Pallas' group order is Vesta's base-field modulus and vice versa (ff/pasta.hpp:92-103)
constexpr curve_ops curve_pallas = curve_row<ff::pallas_gen, ff::vesta_fp_t>();
constexpr curve_ops curve_vesta = curve_row<ff::vesta_gen, ff::pallas_fp_t>();
