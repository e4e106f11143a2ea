// Goldilocks field  p = 2^64 - 2^32 + 1  (the reference's gl64_t, ff/gl64_t.cuh:39-298).
// Memory format of the DATA is the reference's: one plain uint64_t, not Montgomery.  Contract of
// the library's entry points on this field: an input word may be any uint64_t and stands for its value mod p
// (callers such as Plonky2 keep non-canonical words); every output word is canonical (< p).
//
// Representation used by the NTT kernels:
//  * data values travel as "loose" 64-bit residues (any uint64_t, value mod p), from load() on;
//  * every CONSTANT the data is multiplied by (twiddles, coset powers, n^-1) is kept in
//    Montgomery form c' = c * 2^64 mod p, canonical; mul(x, c') = x * c' * 2^-64 = x * c mod p,
//    so products of data and constants are plain again and tables of constants are closed under
//    mul/pow (one() = 2^64 mod p).  The Montgomery reduction for this prime needs no multiply
//    (p^-1 = 1 + 2^32 mod 2^64) and, for a canonical second operand, returns a CANONICAL value
//    for free: with V = a*b < 2^64 * p the exact quotient (V - t*p) / 2^64 lies in (-p, p).
//  * add()/sub() take a loose first and a canonical second operand -- exactly the shape of a
//    radix-2 DIT butterfly (u loose, t = v*w canonical) -- and return loose values; this saves
//    the conditional subtraction on every add/sub.  tight() makes a loose value a legal second
//    operand.  2^64 = 2^32 - 1 =: EPS (mod p), 2^96 = -1 (mod p).
#pragma once
#include "../util/hd.cuh"

struct gl64 {
    typedef uint64_t T;          // storage type in HBM
    static constexpr uint64_t P = 0xffffffff00000001ULL;
    static constexpr uint64_t EPS = 0xffffffffULL;
    static constexpr int MAX_LG = 32;
    static constexpr uint32_t NTT_MAX_LG_R = 12;   // largest sub-NTT per tile (block-tile kernel)
    static constexpr uint32_t NTT_MAX_THREADS = 1024;
    static constexpr uint32_t LG_EPT = 4;          // NTT: elements per thread per register step
    static constexpr int LG_BYTES = 3;

    static HD T canon(T a) { return a >= P ? a - P : a; }
    static HD T tight(T a) { return canon(a); }             // loose -> legal second operand of add/sub
    static HD T load(T a) { return a; }     // memory -> register (accepts non-canonical input)
    static HD T one() { return EPS; }       // 2^64 mod p: the Montgomery form of 1

    // a loose, b canonical -> loose
    static HD T add(T a, T b)
    {
#if defined(__CUDA_ARCH__)
        uint32_t lo, hi, c;
        asm("{ .reg .u32 a0, a1, b0, b1;\n\t"
            "mov.b64 {a0, a1}, %3; mov.b64 {b0, b1}, %4;\n\t"
            "add.cc.u32 %0, a0, b0; addc.cc.u32 %1, a1, b1; addc.u32 %2, 0, 0;\n\t"
            "neg.s32 %2, %2;\n\t"                        // 0 or 0xffffffff == EPS
            "add.cc.u32 %0, %0, %2; addc.u32 %1, %1, 0; }"
            : "=r"(lo), "=r"(hi), "=r"(c) : "l"(a), "l"(b));
        return ((T)hi << 32) | lo;
#else
        T s = a + b;
        return s < a ? s + EPS : s;           // wrapped: +2^64 == +EPS; cannot wrap twice as b < p
#endif
    }
    // a loose, b canonical -> loose
    static HD T sub(T a, T b)
    {
#if defined(__CUDA_ARCH__)
        uint32_t lo, hi, c;
        asm("{ .reg .u32 a0, a1, b0, b1;\n\t"
            "mov.b64 {a0, a1}, %3; mov.b64 {b0, b1}, %4;\n\t"
            "sub.cc.u32 %0, a0, b0; subc.cc.u32 %1, a1, b1; subc.u32 %2, 0, 0;\n\t"   // 0 or EPS
            "sub.cc.u32 %0, %0, %2; subc.u32 %1, %1, 0; }"
            : "=r"(lo), "=r"(hi), "=r"(c) : "l"(a), "l"(b));
        return ((T)hi << 32) | lo;
#else
        T d = a - b;
        return a < b ? d - EPS : d;           // borrowed: -2^64 == -EPS; cannot borrow twice as b < p
#endif
    }
    // (hi:lo) * 2^-64 mod p, hi:lo < 2^64 * p  ->  canonical
    static HD T mont_reduce(T lo, T hi)
    {
        // t = lo * p^-1 mod 2^64 = lo + (lo << 32);  result = hi - ceil(t*p / 2^64) (+p if negative),
        // written with wrapping arithmetic
        T t = lo + (lo << 32);
        T e = t < lo;
        T b = t - (t >> 32) - e;
        T r = hi - b;
        return hi < b ? r - EPS : r;
    }
    // loose x canonical (Montgomery-form constant) -> canonical, = a * b * 2^-64 mod p
    static HD T mul(T a, T b)
    {
#if defined(__CUDA_ARCH__)
        // 128-bit product (ptxas fuses the mad.lo.cc/madc.hi pairs into IMAD.WIDE.U32), then the
        // multiplication-free Montgomery step above on 32-bit halves
        uint32_t s0, s1;
        asm("{ .reg .u32 a0, a1, b0, b1, r0, r1, r2, r3, e, m, x1, y0, y1;\n\t"
            "mov.b64 {a0, a1}, %2; mov.b64 {b0, b1}, %3;\n\t"
            "mul.lo.u32 r0, a0, b0; mul.hi.u32 r1, a0, b0;\n\t"
            "mad.lo.cc.u32 r1, a0, b1, r1; madc.hi.u32 r2, a0, b1, 0;\n\t"
            "mad.lo.cc.u32 r1, a1, b0, r1; madc.hi.cc.u32 r2, a1, b0, r2; addc.u32 r3, 0, 0;\n\t"
            "mad.lo.cc.u32 r2, a1, b1, r2; madc.hi.u32 r3, a1, b1, r3;\n\t"
            "add.cc.u32 x1, r1, r0; addc.u32 e, 0, 0;\n\t"              // t = (x1:r0), carry e
            "sub.cc.u32 y0, r0, x1; subc.u32 y1, x1, 0;\n\t"            // b = t - (t >> 32) - e
            "sub.cc.u32 y0, y0, e;  subc.u32 y1, y1, 0;\n\t"
            "sub.cc.u32 %0, r2, y0; subc.cc.u32 %1, r3, y1; subc.u32 m, 0, 0;\n\t"   // hi - b, m = 0 / EPS
            "sub.cc.u32 %0, %0, m; subc.u32 %1, %1, 0; }"
            : "=r"(s0), "=r"(s1) : "l"(a), "l"(b));
        return ((T)s1 << 32) | s0;
#else
        unsigned __int128 x = (unsigned __int128)a * b;
        return mont_reduce((T)x, (T)(x >> 64));
#endif
    }
    // plain product of two words in the data domain: any a, b -> canonical a * b mod p
    // (2^64 = EPS, 2^96 = -1: hi:lo = lo + hi_lo * EPS - hi_hi); used where BOTH operands are data
    // (prefix products, batch inversion), the NTT never needs it
    static HD T mul_plain(T a, T b)
    {
#if defined(__CUDA_ARCH__)
        const T lo = a * b, hi = __umul64hi(a, b);
#else
        const unsigned __int128 x = (unsigned __int128)a * b;
        const T lo = (T)x, hi = (T)(x >> 64);
#endif
        const T hh = hi >> 32, hl = hi & EPS;
        T t0 = lo - hh;
        if (lo < hh) t0 -= EPS;               // borrowed 2^64 = EPS (mod p); t0 >= 2^64 - 2^32 here
        const T t1 = (hl << 32) - hl;         // hl * EPS <= 2^64 - 2^33 + 1
        T r = t0 + t1;
        if (r < t1) r += EPS;                 // wrapped: r < t1, so r + EPS cannot wrap again
        return canon(r);
    }
    static HD T to_mont(T a) { return mul(canon(a), 0xfffffffe00000001ULL); }   // * 2^128 mod p
    static HD T pow(T b, uint64_t e)
    {
        T r = one();
        b = canon(b);
        for (; e; e >>= 1, b = mul(b, b))
            if (e & 1) r = mul(r, b);
        return r;
    }
    // parameters: ntt/parameters/goldilocks.h:84-160 (default, non-PLONKY2 branch):
    // group_gen = 7, w_(2^32) = 7^((p-1)/2^32) = 0x185629dcda58878c; the constants below are these
    // values times 2^64 mod p (tests/test_params_pin.py pins the plain values, tests/test_emu.py
    // the Montgomery forms)
    static HD T group_gen() { return 0x6fffffff9ULL; }
    static HD T root_of_unity_max() { return 0xda58878b0d514e98ULL; }   // order 2^32
    static HD T inv(T a) { return pow(a, P - 2); }
};
