/*
 * oracle/ntt.h -- TEST INFRASTRUCTURE ONLY (CPU oracle).
 *
 * The reference has NO host NTT (SURVEY.md section 8c); its own tests pin
 * Goldilocks / BabyBear results only by self-consistency
 * (poc/ntt-cuda/tests/ntt.rs:9-79) and 256-bit fields against arkworks.
 * This file therefore restates the DEFINITION the reference's device code
 * implements, with the reference's parameters:
 *   X[k] = sum_j x[j] * w^(j*k),  w = forward_roots_of_unity[lg_n]
 *   inverse: w^-1 and a final * domain_size_inverse[lg_n]   (= 2^-lg_n)
 *   coset:   forward multiplies x[j] by group_gen^j first; inverse multiplies
 *            the result by group_gen^-j last     (ntt/ntt.cuh:196-209,
 *            ntt/kernels.cu:131-153)
 *   orders:  NN natural->natural, NR natural->bit-reversed, RN bit-reversed->natural;
 *            RR is, in the reference, GS on natural input followed by bit_rev, i.e. the SAME
 *            transform as NN (ntt/ntt.cuh:186-189,211-212; poc/ntt-cuda/tests/ntt.rs:28-30
 *            asserts NN == RR), with bit-reversed coset exponents.  ORACLE_BB (4) is the strict
 *            bit-reversed-in / bit-reversed-out transform (an extension, not a reference order).
 *            Pinned by tests/golden/ntt_ref_gpu.npz (the reference's own CUDA kernels).
 * Root conventions (derived, and checked against the ntt/parameters headers by
 * tests/test_params_pin.py):
 *   Goldilocks  w_2^32 = 7^((p-1)/2^32), group_gen = 7   (goldilocks.h:84-160, default branch)
 *   BabyBear    w_2^27 = 137,            group_gen = 3   (baby_bear.h:76-143, default branch)
 *               memory words are Montgomery residues (R = 2^32); by linearity the
 *               transform acts on the raw words with the true-valued roots.
 */
#ifndef ORACLE_NTT_H
#define ORACLE_NTT_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

enum { ORACLE_NN = 0, ORACLE_NR = 1, ORACLE_RN = 2, ORACLE_RR = 3, ORACLE_BB = 4 };

/* in place; direction 0 forward / 1 inverse; type 0 standard / 1 coset;
 * algo 0 fast radix-2 (nthreads>1 uses pthreads), 1 O(n^2) definition */
int oracle_ntt_gl64(uint64_t *inout, unsigned lg_n, int order, int direction, int type,
                    int algo, int nthreads);
int oracle_ntt_bb31(uint32_t *inout, unsigned lg_n, int order, int direction, int type,
                    int algo, int nthreads);

/* 256-bit Montgomery fields: field_id 1 = BLS12-381 fr, 2 = Pallas base field, 3 = Vesta base
 * field; data = n x 4 64-bit limbs, Montgomery residues; in place */
int oracle_ntt_ff(int field_id, uint64_t *data, unsigned lg_n, int order, int direction, int type, int algo);

uint64_t oracle_gl64_root(unsigned lg_n, int inverse);
uint32_t oracle_bb31_root(unsigned lg_n, int inverse);   /* true value, not Montgomery */
uint64_t oracle_gl64_mul(uint64_t a, uint64_t b);

#ifdef __cplusplus
}
#endif
#endif
