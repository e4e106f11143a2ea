// Precomputed fixed-base tables (Config::copies > 1, msm_core.cuh): copy k of point P_i is
// 2^(c*V*k) * P_i, stored copy-major as packed affine rows, row k*N + i.  Copy 0 is the input.
//
//   double     thread = one point of a chunk: c*V XYZZ doublings per copy, copies 1..K-1 kept as
//              XYZZ with their ZZZ (one where the point is infinity: a zero must not enter the product)
//   invert     the ZZZ of the chunk inverted together (pair_invert_body, Montgomery's trick)
//   normalise  thread = one (copy, point): u = 1/ZZZ, x = X (ZZ u)^2, y = Y u; infinity stays (0, 0)
//
// Every body is per-thread (HD: the CPU single-stepper in tests/emu/msm_precomputed_emu.cpp runs
// the same code).
#pragma once
#include "msm_pair.cuh"

namespace msm {

// point first + i of the packed rows -> copies 1..copies-1 at xyzz[(k-1) n + i], their ZZZ at zzz[...]
template<class F>
HD void table_double_body(const uint32_t* packed, size_t first, uint32_t n, uint32_t steps, uint32_t copies,
                          uint32_t* xyzz, uint32_t* zzz, uint32_t i)
{
    const ec::affine_t<F> p = load_point<F>(packed + first * 2 * F::N, i);
    ec::xyzz_t<F> acc;
    if (p.is_inf()) acc.set_inf();
    else acc.set_affine(p);
    for (uint32_t k = 1; k < copies; k++) {
        for (uint32_t s = 0; s < steps; s++) acc.dbl_hot();
        const size_t slot = (size_t)(k - 1) * n + i;
        store_bucket<F>(xyzz, slot, acc);
        pair_store_f<F>(zzz + slot * F::N, acc.is_inf() ? F::one() : acc.ZZZ);
    }
}

// XYZZ point `slot` of the scratch and its inverted ZZZ -> packed affine row: u = 1/ZZZ,
// x = X (ZZ u)^2, y = Y u; infinity -> (0, 0).  Shared by the table build and scale_points
// (msm_scale.cuh).
template<class F>
HD void normalize_to_row(const uint32_t* xyzz, const uint32_t* zzz_inv, uint32_t slot, uint32_t* row)
{
    const ec::xyzz_t<F> acc = load_bucket<F>(xyzz, slot);
    if (acc.is_inf()) {
        pair_store_f<F>(row, F::zero());
        pair_store_f<F>(row + F::N, F::zero());
        return;
    }
    const F u = pair_load_f<F>(zzz_inv + (size_t)slot * F::N);
    const F t = acc.ZZ * u;                             // 1 / Z
    pair_store_f<F>(row, acc.X * t.sqr());
    pair_store_f<F>(row + F::N, acc.Y * u);
}

// slot = (k-1) n + i of the chunk [first, first + n) -> packed affine row k * npoints + first + i
template<class F>
HD void table_normalize_body(const uint32_t* xyzz, const uint32_t* zzz_inv, size_t npoints, size_t first,
                             uint32_t n, uint32_t* table, uint32_t slot)
{
    const uint32_t k = slot / n + 1, i = slot - (k - 1) * n;
    normalize_to_row<F>(xyzz, zzz_inv, slot, table + ((size_t)k * npoints + first + i) * 2 * F::N);
}

}  // namespace msm
