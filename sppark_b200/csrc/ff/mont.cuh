// N x 32-bit Montgomery prime field, R = 2^(32N).
//
// Same memory format as the reference's mont_t (ff/mont_t.cuh:33-44: `uint32_t even[n]`,
// little-endian limbs, Montgomery form), so fp/fr/affine/xyzz buffers are ABI-compatible.
// The arithmetic is this library's own:
//   * multiplication is one fused CIOS ladder over two accumulator files E (pairs at even
//     limb positions) and O (pairs at odd positions).  Every 32x32 product is a single
//     mad.lo.cc/madc.hi.cc pair that ptxas fuses into IMAD.WIDE.U32(.X), all pairs of one
//     row form one carry chain, and the cross-file carry at the vanishing limb is tracked as
//     a 2-bit integer instead of being rippled.  Modulus limbs are compile-time constants and
//     become immediates in SASS.
//   * the portable branch (no __CUDA_ARCH__) is the same ladder on uint64_t, used by the CPU
//     single-stepper in tests/emu and for host-side constants only.
#pragma once
#include "../util/hd.cuh"

namespace ff {

#if defined(__CUDA_ARCH__)
namespace ptx {
DEV void mad_lo_cc(uint32_t& d, uint32_t a, uint32_t b, uint32_t c)
{   asm volatile("mad.lo.cc.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));   }
DEV void madc_lo_cc(uint32_t& d, uint32_t a, uint32_t b, uint32_t c)
{   asm volatile("madc.lo.cc.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));   }
DEV void madc_hi_cc(uint32_t& d, uint32_t a, uint32_t b, uint32_t c)
{   asm volatile("madc.hi.cc.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));   }
DEV void addc(uint32_t& d, uint32_t a, uint32_t b)
{   asm volatile("addc.u32 %0, %1, %2;" : "=r"(d) : "r"(a), "r"(b));   }
DEV void add_cc(uint32_t& d, uint32_t a, uint32_t b)
{   asm volatile("add.cc.u32 %0, %1, %2;" : "=r"(d) : "r"(a), "r"(b));   }
DEV void addc_cc(uint32_t& d, uint32_t a, uint32_t b)
{   asm volatile("addc.cc.u32 %0, %1, %2;" : "=r"(d) : "r"(a), "r"(b));   }
DEV void sub_cc(uint32_t& d, uint32_t a, uint32_t b)
{   asm volatile("sub.cc.u32 %0, %1, %2;" : "=r"(d) : "r"(a), "r"(b));   }
DEV void subc_cc(uint32_t& d, uint32_t a, uint32_t b)
{   asm volatile("subc.cc.u32 %0, %1, %2;" : "=r"(d) : "r"(a), "r"(b));   }
DEV void subc(uint32_t& d, uint32_t a, uint32_t b)
{   asm volatile("subc.u32 %0, %1, %2;" : "=r"(d) : "r"(a), "r"(b));   }
}  // namespace ptx
#endif

// C supplies: static constexpr int N; constexpr accessors P(i), ONE(i), RR(i); M0.
template<class C>
struct mont_t {
    static constexpr int N = C::N;
    uint32_t l[N];

    static HD mont_t zero()
    {
        mont_t r;
#pragma unroll
        for (int i = 0; i < N; i++) r.l[i] = 0;
        return r;
    }
    static HD mont_t one()
    {
        mont_t r;
#pragma unroll
        for (int i = 0; i < N; i++) r.l[i] = C::ONE(i);
        return r;
    }
    static HD mont_t rr()
    {
        mont_t r;
#pragma unroll
        for (int i = 0; i < N; i++) r.l[i] = C::RR(i);
        return r;
    }
    HD bool is_zero() const
    {
        uint32_t acc = 0;
#pragma unroll
        for (int i = 0; i < N; i++) acc |= l[i];
        return acc == 0;
    }
    friend HD bool operator==(const mont_t& a, const mont_t& b)
    {
        uint32_t acc = 0;
#pragma unroll
        for (int i = 0; i < N; i++) acc |= a.l[i] ^ b.l[i];
        return acc == 0;
    }

    // r = a - p if a >= p else a        (a < 2p)
    static HD mont_t final_sub(const mont_t& a, uint32_t top_carry = 0)
    {
        mont_t r;
#if defined(__CUDA_ARCH__)
        uint32_t t[N], borrow;
        ptx::sub_cc(t[0], a.l[0], C::P(0));
#pragma unroll
        for (int i = 1; i < N; i++) ptx::subc_cc(t[i], a.l[i], C::P(i));
        ptx::subc(borrow, top_carry, 0);          // 0 -> a >= p (take t), 0xffffffff -> keep a
#pragma unroll
        for (int i = 0; i < N; i++) r.l[i] = borrow ? a.l[i] : t[i];
#else
        uint32_t t[N];
        int64_t br = 0;
        for (int i = 0; i < N; i++) {
            int64_t d = (int64_t)a.l[i] - C::P(i) + br;
            t[i] = (uint32_t)d;
            br = d >> 32;
        }
        br += top_carry;
        for (int i = 0; i < N; i++) r.l[i] = br < 0 ? a.l[i] : t[i];
#endif
        return r;
    }

    friend HD mont_t operator+(const mont_t& a, const mont_t& b)
    {
        mont_t s;
        uint32_t carry;
#if defined(__CUDA_ARCH__)
        ptx::add_cc(s.l[0], a.l[0], b.l[0]);
#pragma unroll
        for (int i = 1; i < N; i++) ptx::addc_cc(s.l[i], a.l[i], b.l[i]);
        ptx::addc(carry, 0, 0);
#else
        uint64_t c = 0;
        for (int i = 0; i < N; i++) {
            c += (uint64_t)a.l[i] + b.l[i];
            s.l[i] = (uint32_t)c;
            c >>= 32;
        }
        carry = (uint32_t)c;
#endif
        return final_sub(s, carry);
    }

    friend HD mont_t operator-(const mont_t& a, const mont_t& b)
    {
        mont_t d;
#if defined(__CUDA_ARCH__)
        uint32_t borrow;
        ptx::sub_cc(d.l[0], a.l[0], b.l[0]);
#pragma unroll
        for (int i = 1; i < N; i++) ptx::subc_cc(d.l[i], a.l[i], b.l[i]);
        ptx::subc(borrow, 0, 0);                  // 0 or 0xffffffff
        ptx::add_cc(d.l[0], d.l[0], C::P(0) & borrow);
#pragma unroll
        for (int i = 1; i < N - 1; i++) ptx::addc_cc(d.l[i], d.l[i], C::P(i) & borrow);
        ptx::addc(d.l[N - 1], d.l[N - 1], C::P(N - 1) & borrow);
#else
        int64_t br = 0;
        for (int i = 0; i < N; i++) {
            int64_t x = (int64_t)a.l[i] - b.l[i] + br;
            d.l[i] = (uint32_t)x;
            br = x >> 32;
        }
        if (br) {
            uint64_t c = 0;
            for (int i = 0; i < N; i++) {
                c += (uint64_t)d.l[i] + C::P(i);
                d.l[i] = (uint32_t)c;
                c >>= 32;
            }
        }
#endif
        return d;
    }

    HD mont_t neg() const { return is_zero() ? *this : zero() - *this; }
    HD mont_t cneg(bool flag) const { return flag ? neg() : *this; }
    HD mont_t dbl() const { return *this + *this; }

    // ---- Montgomery product a*b*R^-1 mod p ------------------------------------------
#if defined(__CUDA_ARCH__)
    // one row: acc(coords i..i+N+1) += x * v[0..N-1] placed at coord i.  Products with even
    // j go to the file whose pairs start at coord parity(i), odd j to the other one.
    template<int I, class V>
    static DEV void row(uint32_t (&E)[2 * N + 2], uint32_t (&O)[2 * N + 2], uint32_t x, const V& v)
    {
        constexpr bool even_row = (I & 1) == 0;
        uint32_t (&A1)[2 * N + 2] = even_row ? E : O;      // receives even j, pairs at (I+j, I+j+1)
        uint32_t (&A2)[2 * N + 2] = even_row ? O : E;      // receives odd j
        ptx::mad_lo_cc(A1[I], x, v[0], A1[I]);
        ptx::madc_hi_cc(A1[I + 1], x, v[0], A1[I + 1]);
#pragma unroll
        for (int j = 2; j < N; j += 2) {
            ptx::madc_lo_cc(A1[I + j], x, v[j], A1[I + j]);
            ptx::madc_hi_cc(A1[I + j + 1], x, v[j], A1[I + j + 1]);
        }
        ptx::addc(A1[I + N], A1[I + N], 0);
        ptx::mad_lo_cc(A2[I + 1], x, v[1], A2[I + 1]);
        ptx::madc_hi_cc(A2[I + 2], x, v[1], A2[I + 2]);
#pragma unroll
        for (int j = 3; j < N; j += 2) {
            ptx::madc_lo_cc(A2[I + j], x, v[j], A2[I + j]);
            ptx::madc_hi_cc(A2[I + j + 1], x, v[j], A2[I + j + 1]);
        }
        ptx::addc(A2[I + N + 1], A2[I + N + 1], 0);
    }

    struct modulus_view {
        DEV uint32_t operator[](int j) const { return C::P(j); }
    };

    template<int I>
    static DEV void rows(uint32_t (&E)[2 * N + 2], uint32_t (&O)[2 * N + 2], uint32_t& c,
                         const mont_t& a, const mont_t& b)
    {
        if constexpr (I < N) {
            row<I>(E, O, a.l[I], b.l);
            uint32_t m = (E[I] + O[I] + c) * C::M0;
            row<I>(E, O, m, modulus_view());
            // limb I of the running total is now 0 mod 2^32; its carry moves up as an integer
            uint64_t s = (uint64_t)E[I] + O[I] + c;
            c = (uint32_t)(s >> 32);
            rows<I + 1>(E, O, c, a, b);
        }
    }

    // a*b - c*d in the same ladder: step I adds the rows a_I * b and c_I * dn, dn = p - d, then
    // reduces limb I exactly as rows<> does (k is the running carry).  c*dn = -c*d mod p.  a_I and
    // c_I die with their rows.
    template<int I>
    static DEV void msub_rows(uint32_t (&E)[2 * N + 2], uint32_t (&O)[2 * N + 2], uint32_t& k,
                              const mont_t& a, const mont_t& b, const mont_t& c, const mont_t& dn)
    {
        if constexpr (I < N) {
            row<I>(E, O, a.l[I], b.l);
            row<I>(E, O, c.l[I], dn.l);
            uint32_t m = (E[I] + O[I] + k) * C::M0;
            row<I>(E, O, m, modulus_view());
            uint64_t s = (uint64_t)E[I] + O[I] + k;
            k = (uint32_t)(s >> 32);
            msub_rows<I + 1>(E, O, k, a, b, c, dn);
        }
    }
#endif

    friend HD mont_t operator*(const mont_t& a, const mont_t& b) { return mul_inline(a, b); }

    // mul_shared / sqr_shared / msub_shared: ONE copy each per kernel, called (not inlined) from
    // the hot loop.  The unrolled ladder is ~450 instructions and a mixed add has ten products;
    // inlining all of them overflows the instruction cache (no_instruction was the top stall
    // reason before the split, measured on an earlier GPU).  Only called from code that is
    // itself inlined into the kernel, so the call depth is one.
#if defined(__CUDA_ARCH__)
    // ---- double-width arithmetic for the hot loop -----------------------------------------
    // Products kept unreduced (2N limbs), so that a*b can be split Karatsuba-style and reduced in
    // a separate pass.  That trades wide multiplies (the IMAD.WIDE pipe is the busy one in the
    // MSM) for adds and the extra pass; it is compiled out by default (SPPARK_B200_KARATSUBA): on
    // H100 it is slower than the fused ladder in the BLS12-381 G1 hot loop (DESIGN.md section 7.2).
    // The squaring and a*b - c*d instead stay in the fused ladder (sqr_inline, msub_inline).
    struct wide_t { uint32_t l[2 * N]; };

    // acc += x * v[0..W) at limb position I; even j into the file whose pairs sit at parity(I).
    // The carry out of each file's chain lands one limb above that file's last pair, which
    // depends on the parity of W.
    template<int I, int W, class V>
    static DEV void row_w(uint32_t* E, uint32_t* O, uint32_t x, const V& v)
    {
        uint32_t* A1 = (I & 1) == 0 ? E : O;
        uint32_t* A2 = (I & 1) == 0 ? O : E;
        ptx::mad_lo_cc(A1[I], x, v[0], A1[I]);
        ptx::madc_hi_cc(A1[I + 1], x, v[0], A1[I + 1]);
#pragma unroll
        for (int j = 2; j < W; j += 2) {
            ptx::madc_lo_cc(A1[I + j], x, v[j], A1[I + j]);
            ptx::madc_hi_cc(A1[I + j + 1], x, v[j], A1[I + j + 1]);
        }
        ptx::addc(A1[I + W + (W & 1)], A1[I + W + (W & 1)], 0);
        ptx::mad_lo_cc(A2[I + 1], x, v[1], A2[I + 1]);
        ptx::madc_hi_cc(A2[I + 2], x, v[1], A2[I + 2]);
#pragma unroll
        for (int j = 3; j < W; j += 2) {
            ptx::madc_lo_cc(A2[I + j], x, v[j], A2[I + j]);
            ptx::madc_hi_cc(A2[I + j + 1], x, v[j], A2[I + j + 1]);
        }
        ptx::addc(A2[I + W + 1 - (W & 1)], A2[I + W + 1 - (W & 1)], 0);
    }
    template<int I, int W>
    static DEV void mul_rows_w(uint32_t* E, uint32_t* O, const uint32_t* a, const uint32_t* b)
    {
        if constexpr (I < W) {
            row_w<I, W>(E, O, a[I], b);
            mul_rows_w<I + 1, W>(E, O, a, b);
        }
    }
    // t[0..2W) = a[0..W) * b[0..W)
    template<int W>
    static DEV void mul_wide_w(uint32_t* t, const uint32_t* a, const uint32_t* b)
    {
        uint32_t E[2 * W + 2], O[2 * W + 2];
#pragma unroll
        for (int i = 0; i < 2 * W + 2; i++) E[i] = O[i] = 0;
        mul_rows_w<0, W>(E, O, a, b);
        ptx::add_cc(t[0], E[0], O[0]);
#pragma unroll
        for (int i = 1; i < 2 * W - 1; i++) ptx::addc_cc(t[i], E[i], O[i]);
        ptx::addc(t[2 * W - 1], E[2 * W - 1], O[2 * W - 1]);
    }

    // |x - y| over W limbs, returns 1 if x < y
    template<int W>
    static DEV uint32_t abs_diff_w(uint32_t* d, const uint32_t* x, const uint32_t* y)
    {
        uint32_t borrow;
        ptx::sub_cc(d[0], x[0], y[0]);
#pragma unroll
        for (int i = 1; i < W; i++) ptx::subc_cc(d[i], x[i], y[i]);
        ptx::subc(borrow, 0, 0);                      // 0 or 0xffffffff
        // conditional two's-complement negate: (d ^ borrow) - borrow
        ptx::sub_cc(d[0], d[0] ^ borrow, borrow);
#pragma unroll
        for (int i = 1; i < W - 1; i++) ptx::subc_cc(d[i], d[i] ^ borrow, borrow);
        ptx::subc(d[W - 1], d[W - 1] ^ borrow, borrow);
        return borrow & 1;
    }

    // full product, one level of (subtractive) Karatsuba when N is a multiple of 4:
    //   a*b = z0 + (z0 + z2 + s*|a0-a1|*|b1-b0|) * 2^(32H) + z2 * 2^(64H),  H = N/2
    // three H x H products (3*H^2 wide multiplies) instead of N^2
    static DEV wide_t mul_wide(const mont_t& a, const mont_t& b)
    {
        wide_t t;
#if defined(SPPARK_B200_KARATSUBA)
        constexpr bool karatsuba = N % 4 == 0 && N >= 8;
#else
        constexpr bool karatsuba = false;   // off: slower on H100 on every curve (DESIGN.md section 7.2)
#endif
        if constexpr (karatsuba) {
            // Built in place in t: the differences first (a and b die with the two half products),
            // then z0 | z2 in t, zm, and the middle term added into t as three carry chains whose
            // carries out of limb 3H collect in one word.  Live at the peak: t, zm and half of z0.
            constexpr int H = N / 2;
            uint32_t da[H], db[H], zm[2 * H], z0h[H], top, cf;
            const uint32_t neg = 0u - (abs_diff_w<H>(da, a.l, a.l + H) ^ abs_diff_w<H>(db, b.l + H, b.l));
            mul_wide_w<H>(t.l, a.l, b.l);                         // z0 = a0*b0
            mul_wide_w<H>(t.l + 2 * H, a.l + H, b.l + H);         // z2 = a1*b1
            mul_wide_w<H>(zm, da, db);                            // |a0 - a1| * |b1 - b0|
#pragma unroll
            for (int i = 0; i < H; i++) z0h[i] = t.l[H + i];
            // += z2 << 32H: limb 2H + i is read before this chain overwrites it
            ptx::add_cc(t.l[H], t.l[H], t.l[2 * H]);
#pragma unroll
            for (int i = 1; i < 2 * H; i++) ptx::addc_cc(t.l[H + i], t.l[H + i], t.l[2 * H + i]);
            ptx::addc(top, 0, 0);
            // += z0 << 32H
            ptx::add_cc(t.l[H], t.l[H], t.l[0]);
#pragma unroll
            for (int i = 1; i < H; i++) ptx::addc_cc(t.l[H + i], t.l[H + i], t.l[i]);
#pragma unroll
            for (int i = 0; i < H; i++) ptx::addc_cc(t.l[2 * H + i], t.l[2 * H + i], z0h[i]);
            ptx::addc(top, top, 0);
            // +-zm << 32H as (zm ^ neg) + (neg & 1), the sign extension neg going into top;
            // the carry-in comes from neg + neg, which carries exactly when neg is all ones
            ptx::add_cc(cf, neg, neg);
#pragma unroll
            for (int i = 0; i < 2 * H; i++) ptx::addc_cc(t.l[H + i], t.l[H + i], zm[i] ^ neg);
            ptx::addc(top, top, neg);                 // in {0, 1, 2}: the middle term is a0*b1 + a1*b0 >= 0
            ptx::add_cc(t.l[3 * H], t.l[3 * H], top);
#pragma unroll
            for (int i = 3 * H + 1; i < 2 * N - 1; i++) ptx::addc_cc(t.l[i], t.l[i], 0);
            ptx::addc(t.l[2 * N - 1], t.l[2 * N - 1], 0);
        } else {
            mul_wide_w<N>(t.l, a.l, b.l);
        }
        return t;
    }

    // a^2 in the fused ladder: step I adds row I of the square, a_I * (a_I, 2a_{I+1}, ..., 2a_{N-1})
    // at limb 2I, then reduces limb I exactly as rows<> does.  The square terms of limb I all come
    // from rows k <= I/2, so they are in place when m_I is formed.  N(N+1)/2 wide multiplies for
    // the square instead of N^2, with the reduction interleaved as in the product.
    // d[j] = limb j of 2a (2a < 2^(32N) because p < 2^(32N)/3, see sqr_inline)
    template<int I>
    static DEV void sqr_rows(uint32_t* E, uint32_t* O, uint32_t& c, const uint32_t* a, const uint32_t* d)
    {
        if constexpr (I < N) {
            if constexpr (I < N - 1) {
                uint32_t v[N - I];                    // a_I, then 2a with limbs 0..I cleared
                v[0] = a[I];
                v[1] = a[I + 1] << 1;
#pragma unroll
                for (int k = 2; k < N - I; k++) v[k] = d[I + k];
                row_w<2 * I, N - I>(E, O, a[I], v);
            } else {                                  // a_{N-1}^2 alone, at an even limb: file E
                ptx::mad_lo_cc(E[2 * I], a[I], a[I], E[2 * I]);
                ptx::madc_hi_cc(E[2 * I + 1], a[I], a[I], E[2 * I + 1]);
                ptx::addc(E[2 * I + 2], E[2 * I + 2], 0);
            }
            uint32_t m = (E[I] + O[I] + c) * C::M0;
            row_w<I, N>(E, O, m, modulus_view());
            uint64_t s = (uint64_t)E[I] + O[I] + c;
            c = (uint32_t)(s >> 32);
            sqr_rows<I + 1>(E, O, c, a, d);
        }
    }
    static DEV mont_t sqr_inline(const mont_t& a)
    {
        // After step I the two files hold less than sum_{k<=I} a_k 2^(32k) * 2a + p 2^(32(I+1)) <
        // 3p 2^(32(I+1)); p < 2^(32N)/3 keeps that below 2^(32(I+N+1)), so no row chain carries
        // out of its last limb (the product ladder needs only p < 2^(32N)/2).  Larger moduli (some
        // scalar fields) square through the product ladder.
        if constexpr (C::P(N - 1) >= 0x55555555u) {
            return mul_inline(a, a);
        } else {
            uint32_t E[2 * N + 2], O[2 * N + 2], d[N], c = 0;
#pragma unroll
            for (int i = 0; i < 2 * N + 2; i++) E[i] = O[i] = 0;
#pragma unroll
            for (int j = 1; j < N; j++) d[j] = __funnelshift_l(a.l[j - 1], a.l[j], 1);
            sqr_rows<0>(E, O, c, a.l, d);
            mont_t r;
            ptx::add_cc(r.l[0], E[N], c);
#pragma unroll
            for (int i = 1; i < N; i++) ptx::addc_cc(r.l[i], E[N + i], 0);
            ptx::add_cc(r.l[0], r.l[0], O[N]);
#pragma unroll
            for (int i = 1; i < N - 1; i++) ptx::addc_cc(r.l[i], r.l[i], O[N + i]);
            ptx::addc(r.l[N - 1], r.l[N - 1], O[2 * N - 1]);
            return final_sub(r);
        }
    }

    // a*b - c*d with one reduction, in the fused ladder (msub_rows): 3N^2 wide multiplies instead of
    // 4N^2.  dn = p - d lies in (0, p] (p when d = 0), so after step I the two files hold less than
    // (b + dn + p) 2^(32(I+1)) < 3p 2^(32(I+1)), below 2^(32(I+N+1)) when p < 2^(32N)/3 (the
    // condition of sqr_inline): no row chain carries out of its last limb.  The result is below
    // (2p^2 + 2^(32N) p) / 2^(32N) < 2p, so one final_sub makes it canonical.  Larger moduli take
    // two product ladders.
    static DEV mont_t msub_inline(const mont_t& a, const mont_t& b, const mont_t& c, const mont_t& d)
    {
        if constexpr (C::P(N - 1) >= 0x55555555u) {
            return mul_inline(a, b) - mul_inline(c, d);
        } else {
            mont_t dn;
            ptx::sub_cc(dn.l[0], C::P(0), d.l[0]);
#pragma unroll
            for (int i = 1; i < N - 1; i++) ptx::subc_cc(dn.l[i], C::P(i), d.l[i]);
            ptx::subc(dn.l[N - 1], C::P(N - 1), d.l[N - 1]);
            uint32_t E[2 * N + 2], O[2 * N + 2], k = 0;
#pragma unroll
            for (int i = 0; i < 2 * N + 2; i++) E[i] = O[i] = 0;
            msub_rows<0>(E, O, k, a, b, c, dn);
            mont_t r;
            ptx::add_cc(r.l[0], E[N], k);
#pragma unroll
            for (int i = 1; i < N; i++) ptx::addc_cc(r.l[i], E[N + i], 0);
            ptx::add_cc(r.l[0], r.l[0], O[N]);
#pragma unroll
            for (int i = 1; i < N - 1; i++) ptx::addc_cc(r.l[i], r.l[i], O[N + i]);
            ptx::addc(r.l[N - 1], r.l[N - 1], O[2 * N - 1]);
            return final_sub(r);
        }
    }

    // Montgomery reduction of t < K*p*2^(32N) (K = 1 for a product):
    // the multiples m_i*p accumulate in their own even/odd files, limb i of the running total is
    // resolved as an integer carry exactly as in the fused ladder
    template<int I>
    static DEV void redc_rows(uint32_t* E, uint32_t* O, uint32_t& c, const wide_t& t)
    {
        if constexpr (I < N) {
            uint32_t m = (t.l[I] + E[I] + O[I] + c) * C::M0;
            row_w<I, N>(E, O, m, modulus_view());
            uint64_t s = (uint64_t)t.l[I] + E[I] + O[I] + c;
            c = (uint32_t)(s >> 32);
            redc_rows<I + 1>(E, O, c, t);
        }
    }
    template<int K>
    static DEV mont_t redc(const wide_t& t)
    {
        uint32_t E[2 * N + 2], O[2 * N + 2], c = 0;
#pragma unroll
        for (int i = 0; i < 2 * N + 2; i++) E[i] = O[i] = 0;
        redc_rows<0>(E, O, c, t);
        mont_t r;
        uint32_t top, k;                              // bit 32N of the sum (3p may exceed 2^(32N))
        ptx::add_cc(r.l[0], t.l[N], c);
#pragma unroll
        for (int i = 1; i < N; i++) ptx::addc_cc(r.l[i], t.l[N + i], 0);
        ptx::addc(top, 0, 0);
        ptx::add_cc(r.l[0], r.l[0], E[N]);
#pragma unroll
        for (int i = 1; i < N; i++) ptx::addc_cc(r.l[i], r.l[i], E[N + i]);
        ptx::addc(k, 0, 0);
        top += k;
        ptx::add_cc(r.l[0], r.l[0], O[N]);
#pragma unroll
        for (int i = 1; i < N; i++) ptx::addc_cc(r.l[i], r.l[i], O[N + i]);
        ptx::addc(k, 0, 0);
        top += k;
        r = final_sub(r, top);
        if constexpr (K > 1) r = final_sub(r);
        return r;
    }

    // the three shared (non-inlined) entry points of the hot loop
    static __device__ __noinline__ mont_t mul_shared(mont_t a, mont_t b)
    {
#if defined(SPPARK_B200_KARATSUBA)
        return redc<1>(mul_wide(a, b));
#else
        return mul_inline(a, b);                      // the fused ladder: fewest live limbs
#endif
    }
    static __device__ __noinline__ mont_t sqr_shared(mont_t a) { return sqr_inline(a); }
    // a*b - c*d with a single reduction
    static __device__ __noinline__ mont_t msub_shared(mont_t a, mont_t b, mont_t c, mont_t d)
    {   return msub_inline(a, b, c, d);   }
#else
    static inline mont_t mul_shared(const mont_t& a, const mont_t& b) { return mul_inline(a, b); }
    static inline mont_t sqr_shared(const mont_t& a) { return mul_inline(a, a); }
    static inline mont_t msub_shared(const mont_t& a, const mont_t& b, const mont_t& c, const mont_t& d)
    {   return mul_inline(a, b) - mul_inline(c, d);   }
#endif

    static HD mont_t mul_inline(const mont_t& a, const mont_t& b)
    {
        mont_t r;
#if defined(__CUDA_ARCH__)
        uint32_t E[2 * N + 2], O[2 * N + 2], c = 0;
#pragma unroll
        for (int i = 0; i < 2 * N + 2; i++) E[i] = O[i] = 0;
        rows<0>(E, O, c, a, b);
        ptx::add_cc(r.l[0], E[N], c);
#pragma unroll
        for (int i = 1; i < N; i++) ptx::addc_cc(r.l[i], E[N + i], 0);
        ptx::add_cc(r.l[0], r.l[0], O[N]);
#pragma unroll
        for (int i = 1; i < N - 1; i++) ptx::addc_cc(r.l[i], r.l[i], O[N + i]);
        ptx::addc(r.l[N - 1], r.l[N - 1], O[2 * N - 1]);
#else
        uint32_t t[N + 2];
        for (int i = 0; i < N + 2; i++) t[i] = 0;
        for (int i = 0; i < N; i++) {
            uint64_t c = 0;
            for (int j = 0; j < N; j++) {
                c += (uint64_t)a.l[j] * b.l[i] + t[j];
                t[j] = (uint32_t)c;
                c >>= 32;
            }
            c += t[N];
            t[N] = (uint32_t)c;
            t[N + 1] = (uint32_t)(c >> 32);
            uint32_t m = t[0] * C::M0;
            c = ((uint64_t)m * C::P(0) + t[0]) >> 32;
            for (int j = 1; j < N; j++) {
                c += (uint64_t)m * C::P(j) + t[j];
                t[j - 1] = (uint32_t)c;
                c >>= 32;
            }
            c += t[N];
            t[N - 1] = (uint32_t)c;
            t[N] = t[N + 1] + (uint32_t)(c >> 32);
        }
        for (int i = 0; i < N; i++) r.l[i] = t[i];
        return final_sub(r, t[N]);
#endif
        return final_sub(r);
    }

    HD mont_t sqr() const { return *this * *this; }

    HD mont_t to_mont() const { return *this * rr(); }
    HD mont_t from_mont() const
    {
        mont_t o = zero();
        o.l[0] = 1;
        return *this * o;
    }
    HD mont_t inv() const               // Fermat; off the hot path (final normalisations only)
    {
        mont_t acc = one(), base = *this;
        uint32_t e[N];
        uint32_t borrow = 2;                          // e = p - 2, with borrow (P(0) may be 1)
        for (int i = 0; i < N; i++) {
            uint32_t pi = C::P(i);
            e[i] = pi - borrow;
            borrow = pi < borrow ? 1 : 0;
        }
        for (int i = N * 32 - 1; i >= 0; i--) {
            acc = acc.sqr();
            if ((e[i / 32] >> (i % 32)) & 1) acc = acc * base;
        }
        return acc;
    }
};

}  // namespace ff
