/*
 * oracle/shim/blst_t.hpp -- TEST INFRASTRUCTURE ONLY.
 *
 * Stand-in for blst's src/blst_t.hpp (crate blst ~0.3.11, not vendored under
 * the reference tree).  It provides exactly the host-field interface the
 * reference's own headers consume (ff/bls12-381.hpp:91-139, ec/*.hpp,
 * msm/pippenger.hpp, msm/pippenger.cuh host side) so that those headers
 * compile UNMODIFIED from where they lie; see oracle/Makefile.
 * Arithmetic: portable word-serial Montgomery multiplication on 64-bit limbs
 * (no blst assembly), so CPU timings taken through this shim are "sppark's
 * algorithm on portable arithmetic".
 */
#pragma once
#include <cstddef>
#include <cstdint>
#include <cstring>

typedef uint64_t limb_t;
typedef limb_t vec256[4];
typedef limb_t vec384[6];
#define TO_LIMB_T(x) x

namespace shim_detail {
typedef unsigned __int128 u128;

template<size_t N> static inline bool geq(const limb_t* a, const limb_t* m)
{
    for (size_t i = N; i--;)
        if (a[i] != m[i])
            return a[i] > m[i];
    return true;
}
template<size_t N> static inline void sub_n(limb_t* a, const limb_t* m)
{
    limb_t br = 0;
    for (size_t i = 0; i < N; i++) {
        u128 t = (u128)a[i] - m[i] - br;
        a[i] = (limb_t)t;
        br = (limb_t)(t >> 64) & 1;
    }
}
template<size_t N> static inline void add_n(limb_t* a, const limb_t* m)
{
    limb_t c = 0;
    for (size_t i = 0; i < N; i++) {
        u128 t = (u128)a[i] + m[i] + c;
        a[i] = (limb_t)t;
        c = (limb_t)(t >> 64);
    }
}
}  // namespace shim_detail

template<size_t NBITS, size_t N, const limb_t* MOD, limb_t M0, const limb_t* RR,
         const limb_t* ONE>
class shim_field_t {
    limb_t v[N];
    typedef shim_detail::u128 u128;

public:
    static const size_t nbits = NBITS;
    static constexpr size_t bit_length() { return NBITS; }
    static const unsigned degree = 1;
    using mem_t = shim_field_t;
    typedef unsigned char pow_t[(NBITS + 7) / 8];

    shim_field_t() {}
    shim_field_t(const limb_t* p) { memcpy(v, p, sizeof(v)); }

    limb_t& operator[](size_t i) { return v[i]; }
    const limb_t& operator[](size_t i) const { return v[i]; }

    static shim_field_t one(bool or_zero = false)
    {
        shim_field_t r;
        for (size_t i = 0; i < N; i++)
            r.v[i] = or_zero ? 0 : ONE[i];
        return r;
    }
    bool is_zero() const
    {
        limb_t a = 0;
        for (size_t i = 0; i < N; i++)
            a |= v[i];
        return a == 0;
    }
    void zero() { memset(v, 0, sizeof(v)); }

    shim_field_t& operator+=(const shim_field_t& b)
    {
        limb_t c = 0;
        for (size_t i = 0; i < N; i++) {
            u128 t = (u128)v[i] + b.v[i] + c;
            v[i] = (limb_t)t;
            c = (limb_t)(t >> 64);
        }
        if (c || shim_detail::geq<N>(v, MOD))
            shim_detail::sub_n<N>(v, MOD);
        return *this;
    }
    friend shim_field_t operator+(shim_field_t a, const shim_field_t& b) { return a += b; }

    shim_field_t& operator-=(const shim_field_t& b)
    {
        limb_t br = 0;
        for (size_t i = 0; i < N; i++) {
            u128 t = (u128)v[i] - b.v[i] - br;
            v[i] = (limb_t)t;
            br = (limb_t)(t >> 64) & 1;
        }
        if (br)
            shim_detail::add_n<N>(v, MOD);
        return *this;
    }
    friend shim_field_t operator-(shim_field_t a, const shim_field_t& b) { return a -= b; }

    shim_field_t& operator<<=(unsigned l)
    {
        while (l--)
            *this += *this;
        return *this;
    }
    friend shim_field_t operator<<(shim_field_t a, unsigned l) { return a <<= l; }

    shim_field_t& cneg(bool flag)
    {
        if (flag && !is_zero()) {
            shim_field_t z;
            z.zero();
            *this = z - *this;
        }
        return *this;
    }

    friend shim_field_t operator*(const shim_field_t& a, const shim_field_t& b)
    {
        limb_t t[N + 2];
        memset(t, 0, sizeof(t));
        for (size_t i = 0; i < N; i++) {
            limb_t c = 0;
            for (size_t j = 0; j < N; j++) {
                u128 x = (u128)a.v[j] * b.v[i] + t[j] + c;
                t[j] = (limb_t)x;
                c = (limb_t)(x >> 64);
            }
            u128 x = (u128)t[N] + c;
            t[N] = (limb_t)x;
            t[N + 1] = (limb_t)(x >> 64);
            limb_t m = t[0] * M0;
            x = (u128)m * MOD[0] + t[0];
            c = (limb_t)(x >> 64);
            for (size_t j = 1; j < N; j++) {
                x = (u128)m * MOD[j] + t[j] + c;
                t[j - 1] = (limb_t)x;
                c = (limb_t)(x >> 64);
            }
            x = (u128)t[N] + c;
            t[N - 1] = (limb_t)x;
            t[N] = t[N + 1] + (limb_t)(x >> 64);
        }
        shim_field_t r;
        memcpy(r.v, t, sizeof(r.v));
        if (t[N] || shim_detail::geq<N>(r.v, MOD))
            shim_detail::sub_n<N>(r.v, MOD);
        return r;
    }
    shim_field_t& operator*=(const shim_field_t& b) { return *this = *this * b; }
    shim_field_t& sqr() { return *this = *this * *this; }
    shim_field_t& operator^=(int p)
    {
        if (p == 2)
            return sqr();
        shim_field_t b = *this;
        for (int i = 1; i < p; i++)
            *this *= b;
        return *this;
    }
    friend shim_field_t operator^(shim_field_t a, int p) { return a ^= p; }

    void to() { *this = *this * shim_field_t(RR); }
    void from()
    {
        shim_field_t o;
        o.zero();
        o.v[0] = 1;
        *this = *this * o;
    }
    void to_scalar(pow_t& s) const
    {
        shim_field_t t = *this;
        t.from();
        memcpy(s, t.v, sizeof(pow_t));
    }
    friend bool operator==(const shim_field_t& a, const shim_field_t& b)
    {
        return memcmp(a.v, b.v, sizeof(a.v)) == 0;
    }
    friend bool operator!=(const shim_field_t& a, const shim_field_t& b) { return !(a == b); }
    friend shim_field_t czero(const shim_field_t& a, int set_z)
    {
        shim_field_t r = a;
        if (set_z)
            r.zero();
        return r;
    }
    static shim_field_t csel(const shim_field_t& a, const shim_field_t& b, int sel_a)
    {
        return sel_a ? a : b;
    }
    shim_field_t reciprocal() const
    {
        limb_t e[N];
        memcpy(e, MOD, sizeof(e));
        e[0] -= 2;
        shim_field_t r = one(), b = *this;
        for (size_t i = 0; i < N * 64; i++) {
            if ((e[i / 64] >> (i % 64)) & 1)
                r *= b;
            b.sqr();
        }
        return r;
    }
    friend shim_field_t operator/(int, const shim_field_t& a) { return a.reciprocal(); }
};

template<size_t NBITS, const limb_t* MOD, limb_t M0, const limb_t* RR, const limb_t* ONE>
using blst_256_t = shim_field_t<NBITS, 4, MOD, M0, RR, ONE>;
template<size_t NBITS, const limb_t* MOD, limb_t M0, const limb_t* RR, const limb_t* ONE>
using blst_384_t = shim_field_t<NBITS, 6, MOD, M0, RR, ONE>;

/* ---- blst C-level vector API (blst src/vect.h, consumed by the host half of
 * ff/bls12-381-fp2.hpp:158-417).  Own portable code, same signatures. ------------------------ */
typedef vec384 vec384x[2];

static inline void vec_copy(void* d, const void* s, size_t n) { memcpy(d, s, n); }
static inline void vec_zero(void* d, size_t n) { memset(d, 0, n); }
static inline bool vec_is_zero(const void* a, size_t n)
{
    const unsigned char* p = (const unsigned char*)a;
    unsigned char acc = 0;
    for (size_t i = 0; i < n; i++) acc |= p[i];
    return acc == 0;
}
static inline bool vec_is_equal(const void* a, const void* b, size_t n) { return memcmp(a, b, n) == 0; }
static inline void vec_select(void* d, const void* a, const void* b, size_t n, bool sel_a)
{   memmove(d, sel_a ? a : b, n);   }

static inline void mul_mont_384(vec384 r, const vec384 a, const vec384 b, const vec384 p, limb_t n0)
{
    typedef shim_detail::u128 u128;
    limb_t t[8] = {0};
    for (size_t i = 0; i < 6; i++) {
        limb_t c = 0;
        for (size_t j = 0; j < 6; j++) {
            u128 x = (u128)a[j] * b[i] + t[j] + c;
            t[j] = (limb_t)x; c = (limb_t)(x >> 64);
        }
        u128 s = (u128)t[6] + c;
        t[6] = (limb_t)s; t[7] = (limb_t)(s >> 64);
        limb_t m = t[0] * n0;
        u128 x = (u128)m * p[0] + t[0];
        c = (limb_t)(x >> 64);
        for (size_t j = 1; j < 6; j++) {
            x = (u128)m * p[j] + t[j] + c;
            t[j - 1] = (limb_t)x; c = (limb_t)(x >> 64);
        }
        s = (u128)t[6] + c;
        t[5] = (limb_t)s; t[6] = t[7] + (limb_t)(s >> 64);
    }
    if (t[6] || shim_detail::geq<6>(t, p)) shim_detail::sub_n<6>(t, p);
    memcpy(r, t, sizeof(vec384));
}
static inline void from_mont_384(vec384 r, const vec384 a, const vec384 p, limb_t n0)
{
    const vec384 one = {1};
    mul_mont_384(r, a, one, p, n0);
}
static inline void add_mod_384(vec384 r, const vec384 a, const vec384 b, const vec384 p)
{
    typedef shim_detail::u128 u128;
    limb_t t[6], c = 0;
    for (size_t i = 0; i < 6; i++) { u128 x = (u128)a[i] + b[i] + c; t[i] = (limb_t)x; c = (limb_t)(x >> 64); }
    if (c || shim_detail::geq<6>(t, p)) shim_detail::sub_n<6>(t, p);
    memcpy(r, t, sizeof(vec384));
}
static inline void sub_mod_384(vec384 r, const vec384 a, const vec384 b, const vec384 p)
{
    typedef shim_detail::u128 u128;
    limb_t t[6], br = 0;
    for (size_t i = 0; i < 6; i++) { u128 x = (u128)a[i] - b[i] - br; t[i] = (limb_t)x; br = (limb_t)(x >> 64) & 1; }
    if (br) shim_detail::add_n<6>(t, p);
    memcpy(r, t, sizeof(vec384));
}
static inline void cneg_mod_384(vec384 r, const vec384 a, bool flag, const vec384 p)
{
    if (flag && !vec_is_zero(a, sizeof(vec384))) {
        const vec384 zero = {0};
        sub_mod_384(r, zero, a, p);
    } else {
        memmove(r, a, sizeof(vec384));
    }
}
static inline void lshift_mod_384(vec384 r, const vec384 a, size_t n, const vec384 p)
{
    vec384 t;
    memcpy(t, a, sizeof(t));
    while (n--) add_mod_384(t, t, t, p);
    memcpy(r, t, sizeof(t));
}
static inline void rshift_mod_384(vec384 r, const vec384 a, size_t n, const vec384 p)
{
    typedef shim_detail::u128 u128;
    limb_t t[6];
    memcpy(t, a, sizeof(t));
    while (n--) {
        limb_t c = 0;
        if (t[0] & 1)
            for (size_t i = 0; i < 6; i++) { u128 x = (u128)t[i] + p[i] + c; t[i] = (limb_t)x; c = (limb_t)(x >> 64); }
        for (size_t i = 0; i < 5; i++) t[i] = (t[i] >> 1) | (t[i + 1] << 63);
        t[5] = (t[5] >> 1) | (c << 63);
    }
    memcpy(r, t, sizeof(t));
}
// ---- the 256-bit members of the same family (ff/alt_bn128-fp2.hpp's host fp2_t calls them directly) ----
namespace shim_detail {
template<size_t N> static inline void mul_mont_n(limb_t* r, const limb_t* a, const limb_t* b, const limb_t* p, limb_t n0)
{
    limb_t t[N + 2] = {0};
    for (size_t i = 0; i < N; i++) {
        limb_t c = 0;
        for (size_t j = 0; j < N; j++) {
            u128 x = (u128)a[j] * b[i] + t[j] + c;
            t[j] = (limb_t)x; c = (limb_t)(x >> 64);
        }
        u128 s = (u128)t[N] + c;
        t[N] = (limb_t)s; t[N + 1] = (limb_t)(s >> 64);
        limb_t m = t[0] * n0;
        u128 x = (u128)m * p[0] + t[0];
        c = (limb_t)(x >> 64);
        for (size_t j = 1; j < N; j++) {
            x = (u128)m * p[j] + t[j] + c;
            t[j - 1] = (limb_t)x; c = (limb_t)(x >> 64);
        }
        s = (u128)t[N] + c;
        t[N - 1] = (limb_t)s; t[N] = t[N + 1] + (limb_t)(s >> 64);
    }
    if (t[N] || geq<N>(t, p)) sub_n<N>(t, p);
    memcpy(r, t, N * sizeof(limb_t));
}
}  // namespace shim_detail
static inline void mul_mont_sparse_256(vec256 r, const vec256 a, const vec256 b, const vec256 p, limb_t n0)
{   shim_detail::mul_mont_n<4>(r, a, b, p, n0);   }
static inline void sqr_mont_sparse_256(vec256 r, const vec256 a, const vec256 p, limb_t n0)
{   shim_detail::mul_mont_n<4>(r, a, a, p, n0);   }
static inline void from_mont_256(vec256 r, const vec256 a, const vec256 p, limb_t n0)
{
    const vec256 one = {1};
    shim_detail::mul_mont_n<4>(r, a, one, p, n0);
}
static inline void add_mod_256(vec256 r, const vec256 a, const vec256 b, const vec256 p)
{
    typedef shim_detail::u128 u128;
    limb_t t[4], c = 0;
    for (size_t i = 0; i < 4; i++) { u128 x = (u128)a[i] + b[i] + c; t[i] = (limb_t)x; c = (limb_t)(x >> 64); }
    if (c || shim_detail::geq<4>(t, p)) shim_detail::sub_n<4>(t, p);
    memcpy(r, t, sizeof(vec256));
}
static inline void sub_mod_256(vec256 r, const vec256 a, const vec256 b, const vec256 p)
{
    typedef shim_detail::u128 u128;
    limb_t t[4], br = 0;
    for (size_t i = 0; i < 4; i++) { u128 x = (u128)a[i] - b[i] - br; t[i] = (limb_t)x; br = (limb_t)(x >> 64) & 1; }
    if (br) shim_detail::add_n<4>(t, p);
    memcpy(r, t, sizeof(vec256));
}
static inline void cneg_mod_256(vec256 r, const vec256 a, bool flag, const vec256 p)
{
    if (flag && !vec_is_zero(a, sizeof(vec256))) {
        const vec256 zero = {0};
        sub_mod_256(r, zero, a, p);
    } else {
        memmove(r, a, sizeof(vec256));
    }
}
static inline void lshift_mod_256(vec256 r, const vec256 a, size_t n, const vec256 p)
{
    vec256 t;
    memcpy(t, a, sizeof(t));
    while (n--) add_mod_256(t, t, t, p);
    memcpy(r, t, sizeof(t));
}
static inline void rshift_mod_256(vec256 r, const vec256 a, size_t n, const vec256 p)
{
    typedef shim_detail::u128 u128;
    limb_t t[4];
    memcpy(t, a, sizeof(t));
    while (n--) {
        limb_t c = 0;
        if (t[0] & 1)
            for (size_t i = 0; i < 4; i++) { u128 x = (u128)t[i] + p[i] + c; t[i] = (limb_t)x; c = (limb_t)(x >> 64); }
        for (size_t i = 0; i < 3; i++) t[i] = (t[i] >> 1) | (t[i + 1] << 63);
        t[3] = (t[3] >> 1) | (c << 63);
    }
    memcpy(r, t, sizeof(t));
}

static inline void add_mod_384x(vec384x r, const vec384x a, const vec384x b, const vec384 p)
{   add_mod_384(r[0], a[0], b[0], p); add_mod_384(r[1], a[1], b[1], p);   }
static inline void sub_mod_384x(vec384x r, const vec384x a, const vec384x b, const vec384 p)
{   sub_mod_384(r[0], a[0], b[0], p); sub_mod_384(r[1], a[1], b[1], p);   }
/* Fp2 = Fp[u]/(u^2+1), schoolbook */
static inline void mul_mont_384x(vec384x r, const vec384x a, const vec384x b, const vec384 p, limb_t n0)
{
    vec384 t0, t1, t2, t3;
    mul_mont_384(t0, a[0], b[0], p, n0);
    mul_mont_384(t1, a[1], b[1], p, n0);
    mul_mont_384(t2, a[0], b[1], p, n0);
    mul_mont_384(t3, a[1], b[0], p, n0);
    sub_mod_384(r[0], t0, t1, p);
    add_mod_384(r[1], t2, t3, p);
}
static inline void sqr_mont_384x(vec384x r, const vec384x a, const vec384 p, limb_t n0)
{   mul_mont_384x(r, a, a, p, n0);   }

static inline void be_bytes_from_limbs(unsigned char* out, const limb_t* in, size_t n)
{
    for (size_t i = 0; i < n; i++) out[n - 1 - i] = (unsigned char)(in[i / 8] >> (8 * (i % 8)));
}
static inline char hex_from_nibble(unsigned char n) { return "0123456789abcdef"[n & 15]; }
