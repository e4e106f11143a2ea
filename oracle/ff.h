/*
 * oracle/ff.h -- TEST INFRASTRUCTURE ONLY (CPU oracle).
 *
 * Portable Montgomery prime-field arithmetic on 64-bit limbs (unsigned
 * __int128 products).  It stands in for the host-side field types the
 * reference takes from third-party code that is NOT vendored under
 * the reference tree:
 *   - blst  src/blst_t.hpp  (crate blst ~0.3.11, poc/msm-cuda/Cargo.toml:24)
 *       -> blst_384_t / blst_256_t, used by ff/bls12-381.hpp:91-139
 *   - semolina pasta_t.hpp  (crate semolina ~0.1.2, poc/ntt-cuda/Cargo.toml:28)
 *       -> pallas_t / vesta_t, used by ff/pasta.hpp:82-103
 * The published algorithm restated here is word-serial Montgomery
 * multiplication (CIOS): t = a*b*R^-1 mod p with R = 2^(64*n).
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg may
 * use anything under oracle/.  The product (sppark_b200/csrc) never does.
 */
#ifndef ORACLE_FF_H
#define ORACLE_FF_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FF_MAX_LIMBS 6

typedef struct {
    int n;                       /* 64-bit limbs: 4 (<=256 bit) or 6 (<=384 bit) */
    int nbits;                   /* bit length of the modulus                    */
    uint64_t p[FF_MAX_LIMBS];    /* modulus, little-endian limbs                  */
    uint64_t m0;                 /* -p^-1 mod 2^64                                */
    uint64_t rr[FF_MAX_LIMBS];   /* R^2 mod p                                     */
    uint64_t one[FF_MAX_LIMBS];  /* R mod p                                       */
} ff_ctx;

typedef struct { uint64_t l[FF_MAX_LIMBS]; } ff_t;

/* Build a context from the modulus alone; m0, RR and ONE are derived, so the
 * tests can cross-check them against the constants the reference hard-codes
 * (ff/bls12-381.hpp:100-139, ff/pasta.hpp:14-50). */
void ff_ctx_init(ff_ctx *c, const uint64_t *p, int n, int nbits);

void ff_mul(const ff_ctx *c, ff_t *r, const ff_t *a, const ff_t *b);
void ff_sqr(const ff_ctx *c, ff_t *r, const ff_t *a);
void ff_add(const ff_ctx *c, ff_t *r, const ff_t *a, const ff_t *b);
void ff_sub(const ff_ctx *c, ff_t *r, const ff_t *a, const ff_t *b);
void ff_neg(const ff_ctx *c, ff_t *r, const ff_t *a);       /* 0 stays 0 */
void ff_to_mont(const ff_ctx *c, ff_t *r, const ff_t *a);    /* a*R       */
void ff_from_mont(const ff_ctx *c, ff_t *r, const ff_t *a);  /* a*R^-1    */
void ff_inv(const ff_ctx *c, ff_t *r, const ff_t *a);        /* Fermat    */
int  ff_is_zero(const ff_ctx *c, const ff_t *a);
int  ff_eq(const ff_ctx *c, const ff_t *a, const ff_t *b);
void ff_set_zero(ff_t *r);
void ff_set_one(const ff_ctx *c, ff_t *r);                   /* Montgomery 1 */

/* the three 255/381-bit primes the hot path uses */
const ff_ctx *ff_bls12_381_fp(void);
const ff_ctx *ff_bls12_381_fr(void);
const ff_ctx *ff_pallas_fp(void);   /* Pallas base field  = Vesta scalar field */
const ff_ctx *ff_vesta_fp(void);    /* Vesta base field   = Pallas scalar field */
const ff_ctx *ff_bn254_fp(void);
const ff_ctx *ff_bn254_fr(void);
const ff_ctx *ff_bls12_377_fp(void);
const ff_ctx *ff_bls12_377_fr(void);

#ifdef __cplusplus
}
#endif
#endif
