// Scalar multiplication of point arrays: out[i] = s_i * P_i as packed affine rows, in chunks of at
// most SCALE_CHUNK points, three steps per chunk (the table build of msm_table.cuh with an arbitrary
// scalar in place of 2^(c*V*k)):
//
//   ladder     thread = one point: the scalar recoded into signed windows of SCALE_WBITS bits (the
//              MSM's Digits, bottom-up with carry), the table j*P, j = 1 .. 2^(w-1), built in XYZZ
//              by mixed additions of P, then per window from the top: w doublings and one addition
//              of +-T[|d| - 1] (none for a zero digit).  XYZZ result and its ZZZ to scratch (one
//              where the result is infinity: a zero must not enter the product)
//   invert     the ZZZ of the chunk inverted together (pair_invert_body, Montgomery's trick)
//   normalise  thread = one point: normalize_to_row, as the table build
//
// The ladder is not constant-time: which additions run, and the table index, follow the digits.
// Every body is per-thread (HD: the CPU single-stepper in tests/emu/msm_scale_emu.cpp runs the same
// code).
#pragma once
#include "msm_table.cuh"

namespace msm {

// 5: 1.8 % faster than 4 on BLS12-381 G1 at 2^20 points (DESIGN.md section 5e), for twice the per-lane table
#ifndef SPPARK_B200_SCALE_WBITS
# define SPPARK_B200_SCALE_WBITS 5
#endif
constexpr uint32_t SCALE_WBITS = SPPARK_B200_SCALE_WBITS;  // signed window width of the ladder
constexpr uint32_t SCALE_TABLE = 1u << (SCALE_WBITS - 1);  // XYZZ entries j*P, j = 1 .. 2^(w-1), per lane
constexpr uint32_t SCALE_MAX_DIGITS = (255 + SCALE_WBITS) / SCALE_WBITS;   // digits_for(255, w)
constexpr size_t SCALE_CHUNK = (size_t)1 << 22;            // points per chunk: 5 * F::N words of scratch each

// point i of `points` times scalar i of `scalars` (SW 32-bit words each, bits from nbits up ignored)
// -> XYZZ at xyzz[i], its ZZZ (one for infinity) at zzz[i]
template<class F, uint32_t SW>
HD void scale_ladder_body(const uint32_t* points, const uint32_t* scalars, uint32_t nbits, uint32_t* xyzz,
                          uint32_t* zzz, uint32_t i)
{
    constexpr uint32_t W = SCALE_WBITS;
    const ec::affine_t<F> p = load_point<F>(points, i);
    ec::xyzz_t<F> acc;
    acc.set_inf();
    if (!p.is_inf()) {
        // the digits bottom-up (the carry runs upwards), consumed top-down: |d| in the low bits, sign in bit 7
        Digits<SW> d(scalars + (size_t)SW * i, nbits);
        const uint32_t nd = digits_for(nbits, W);
        uint8_t dig[SCALE_MAX_DIGITS];
        for (uint32_t w = 0; w < nd; w++) {
            uint32_t bucket, neg;
            dig[w] = d.next(w, W, bucket, neg) ? (uint8_t)((bucket + 1) | (neg << 7)) : 0;
        }
        ec::xyzz_t<F> tab[SCALE_TABLE];
        tab[0].set_affine(p);
        for (uint32_t j = 1; j < SCALE_TABLE; j++) {
            tab[j] = tab[j - 1];
            tab[j].madd(p);
        }
        for (uint32_t w = nd; w-- > 0;) {
            for (uint32_t s = 0; s < W; s++) acc.dbl_hot();        // infinity stays infinity: free at the top
            if (dig[w]) {
                ec::xyzz_t<F> t = tab[(dig[w] & 0x7f) - 1];
                if (dig[w] >> 7) t.Y = t.Y.neg();
                acc.add_hot(t);
            }
        }
    }
    store_bucket<F>(xyzz, i, acc);
    pair_store_f<F>(zzz + (size_t)i * F::N, acc.is_inf() ? F::one() : acc.ZZZ);
}

}  // namespace msm
