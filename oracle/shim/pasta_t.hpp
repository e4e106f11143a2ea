/*
 * oracle/shim/pasta_t.hpp -- TEST INFRASTRUCTURE ONLY.
 *
 * Stand-in for semolina's pasta_t.hpp (crate semolina ~0.1.2, poc/ntt-cuda/Cargo.toml:28; not
 * vendored in the reference tree), which the reference's ff/pasta.hpp:82-84 includes for its
 * HOST-side field types.  It provides the two class names that header expects, pallas_t and
 * vesta_t, on the same portable Montgomery class as oracle/shim/blst_t.hpp, so that
 * ff/pasta.hpp, ec/*.hpp and msm/pippenger.cuh compile UNMODIFIED from where they lie and the
 * reference's own CUDA MSM can be run for the Pasta curves (oracle/ref_msm_g1.cu, oracle/Makefile).
 * Constants: the two Pasta primes and their Montgomery parameters for R = 2^256 (re-derived;
 * tests/test_params_pin.py compares them with the device-side tables of ff/pasta.hpp:12-50).
 */
#pragma once
#include "blst_t.hpp"

namespace pasta_shim {
static const vec256 Pallas_P = {
    TO_LIMB_T(0x992d30ed00000001), TO_LIMB_T(0x224698fc094cf91b),
    TO_LIMB_T(0x0000000000000000), TO_LIMB_T(0x4000000000000000)
};
static const vec256 Pallas_RR = {       /* (1<<512)%P */
    TO_LIMB_T(0x8c78ecb30000000f), TO_LIMB_T(0xd7d30dbd8b0de0e7),
    TO_LIMB_T(0x7797a99bc3c95d18), TO_LIMB_T(0x096d41af7b9cb714)
};
static const vec256 Pallas_ONE = {      /* (1<<256)%P */
    TO_LIMB_T(0x34786d38fffffffd), TO_LIMB_T(0x992c350be41914ad),
    TO_LIMB_T(0xffffffffffffffff), TO_LIMB_T(0x3fffffffffffffff)
};
static const vec256 Vesta_P = {
    TO_LIMB_T(0x8c46eb2100000001), TO_LIMB_T(0x224698fc0994a8dd),
    TO_LIMB_T(0x0000000000000000), TO_LIMB_T(0x4000000000000000)
};
static const vec256 Vesta_RR = {        /* (1<<512)%P */
    TO_LIMB_T(0xfc9678ff0000000f), TO_LIMB_T(0x67bb433d891a16e3),
    TO_LIMB_T(0x7fae231004ccf590), TO_LIMB_T(0x096d41af7ccfdaa9)
};
static const vec256 Vesta_ONE = {       /* (1<<256)%P */
    TO_LIMB_T(0x5b2b3e9cfffffffd), TO_LIMB_T(0x992c350be3420567),
    TO_LIMB_T(0xffffffffffffffff), TO_LIMB_T(0x3fffffffffffffff)
};
typedef blst_256_t<255, Pallas_P, 0x992d30ecffffffffu, Pallas_RR, Pallas_ONE> pallas_mont;
typedef blst_256_t<255, Vesta_P, 0x8c46eb20ffffffffu, Vesta_RR, Vesta_ONE> vesta_mont;
}  // namespace pasta_shim

# if defined(__GNUC__) && !defined(__clang__)
#  pragma GCC diagnostic push
#  pragma GCC diagnostic ignored "-Wsubobject-linkage"
# endif
struct pallas_t : public pasta_shim::pallas_mont {
    using mem_t = pallas_t;
    inline pallas_t() {}
    inline pallas_t(const pasta_shim::pallas_mont& a) : pasta_shim::pallas_mont(a) {}
    template<typename... Ts> constexpr pallas_t(Ts... a) : pasta_shim::pallas_mont{a...} {}
};
struct vesta_t : public pasta_shim::vesta_mont {
    using mem_t = vesta_t;
    inline vesta_t() {}
    inline vesta_t(const pasta_shim::vesta_mont& a) : pasta_shim::vesta_mont(a) {}
    template<typename... Ts> constexpr vesta_t(Ts... a) : pasta_shim::vesta_mont{a...} {}
};
# if defined(__GNUC__) && !defined(__clang__)
#  pragma GCC diagnostic pop
# endif
