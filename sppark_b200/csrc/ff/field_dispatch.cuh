// SPPARK_FIELD_* id (include/sppark_b200.h) -> field type, for the C entry points of the NTT, LDE and
// polynomial blocks: fn(field_tag<F>{}) with F the id's field, the refusal `msg` for any other id.
#pragma once
#include "gl64.cuh"
#include "bb31.cuh"
#include "mont_ntt.cuh"
#include "../util/gpu.cuh"

template<class F> struct field_tag { typedef F type; };

// all seven NTT fields
template<class Fn> RustError with_field(int field, const char* msg, Fn&& fn)
{
    switch (field) {
    case SPPARK_FIELD_GL64: return fn(field_tag<gl64>{});
    case SPPARK_FIELD_BB31: return fn(field_tag<bb31>{});
    case SPPARK_FIELD_BLS12_381_FR: return fn(field_tag<ff::bls12_381_fr_ntt>{});
    case SPPARK_FIELD_PALLAS_FR: return fn(field_tag<ff::pallas_fr_ntt>{});
    case SPPARK_FIELD_VESTA_FR: return fn(field_tag<ff::vesta_fr_ntt>{});
    case SPPARK_FIELD_BN254_FR: return fn(field_tag<ff::bn254_fr_ntt>{});
    case SPPARK_FIELD_BLS12_377_FR: return fn(field_tag<ff::bls12_377_fr_ntt>{});
    default: return rust_err(-(int)cudaErrorInvalidValue, msg);
    }
}

// Goldilocks and BabyBear only: fn is instantiated for the single-word fields alone.  The ids of the
// 256-bit fields get `wide_msg` if there is one, `msg` otherwise
template<class Fn> RustError with_word_field(int field, const char* msg, const char* wide_msg, Fn&& fn)
{
    switch (field) {
    case SPPARK_FIELD_GL64: return fn(field_tag<gl64>{});
    case SPPARK_FIELD_BB31: return fn(field_tag<bb31>{});
    case SPPARK_FIELD_BLS12_381_FR: case SPPARK_FIELD_PALLAS_FR: case SPPARK_FIELD_VESTA_FR:
    case SPPARK_FIELD_BN254_FR: case SPPARK_FIELD_BLS12_377_FR:
        if (wide_msg) return rust_err(-(int)cudaErrorInvalidValue, wide_msg);
        [[fallthrough]];
    default: return rust_err(-(int)cudaErrorInvalidValue, msg);
    }
}
