// Short-Weierstrass (a = 0) point types of the MSM path, ABI-compatible with the reference:
//   affine_t   {X, Y}            infinity = X == Y == 0         (ec/affine_t.hpp:19-72)
//   xyzz_t     {X, Y, ZZZ, ZZ}   infinity = ZZZ == ZZ == 0      (ec/xyzz_t.hpp:16-17,94-101)
//   jacobian_t {X, Y, Z}         infinity = Z == 0              (ec/jacobian_t.hpp:16-58)
// x = X/ZZ, y = Y/ZZZ with ZZ^3 = ZZZ^2.  Formulae: EFD shortw-xyzz madd-2008-s / add-2008-s /
// dbl-2008-s-1 / mdbl-2008-s-1, with the same exceptional-case behaviour as the reference
// (operand at infinity, P+P -> doubling, P+(-P) -> infinity; ec/xyzz_t.hpp:117-200,352-429).
#pragma once
#include "../ff/mont.cuh"

namespace ec {

template<class F> struct affine_t {
    F X, Y;
    HD bool is_inf() const
    {
        uint32_t acc = 0;
#pragma unroll
        for (int i = 0; i < F::N; i++) acc |= X.l[i] | Y.l[i];
        return acc == 0;
    }
};

template<class F> struct jacobian_t {
    F X, Y, Z;
};

template<class F> struct xyzz_t {
    F X, Y, ZZZ, ZZ;

    HD void set_inf()
    {
        X = F::zero(); Y = F::zero(); ZZZ = F::zero(); ZZ = F::zero();
    }
    HD bool is_inf() const
    {
        uint32_t acc = 0;
#pragma unroll
        for (int i = 0; i < F::N; i++) acc |= ZZZ.l[i] | ZZ.l[i];
        return acc == 0;
    }
    HD void set_affine(const affine_t<F>& p)        // p must not be infinity
    {
        X = p.X; Y = p.Y; ZZZ = F::one(); ZZ = F::one();
    }

    // doubling of an affine point (mdbl-2008-s-1, a = 0)
    HD_NOINLINE void set_double_of(const affine_t<F>& p)
    {
        F U = p.Y.dbl();
        F V = U.sqr();
        F W = U * V;
        F S = p.X * V;
        F M = p.X.sqr();
        M = M.dbl() + M;
        F X3 = M.sqr() - S - S;
        Y = M * (S - X3) - W * p.Y;
        X = X3;
        ZZ = V;
        ZZZ = W;
    }

    // *this += p2  (p2 affine, Y already sign-adjusted by the caller).  8M + 2S.
    // This is the hot loop of the MSM: its ten products go through F::mul_shared.
    HD void madd(const affine_t<F>& p2)
    {
        if (p2.is_inf()) return;
        if (is_inf()) { set_affine(p2); return; }
        F P = F::mul_shared(p2.X, ZZ) - X;          // U2 - X1
        F R = F::mul_shared(p2.Y, ZZZ) - Y;         // S2 - Y1
        if (P.is_zero()) {
            if (R.is_zero()) set_double_of(p2);
            else set_inf();
            return;
        }
        F PP = F::sqr_shared(P);
        F PPP = F::mul_shared(P, PP);
        F Q = F::mul_shared(X, PP);
        F X3 = F::sqr_shared(R) - PPP - Q - Q;
        Y = F::msub_shared(R, Q - X3, Y, PPP);      // R*(Q-X3) - Y1*PPP, one reduction
        X = X3;
        ZZ = F::mul_shared(ZZ, PP);
        ZZZ = F::mul_shared(ZZZ, PPP);
    }

    // in-place doubling (dbl-2008-s-1, a = 0); infinity stays infinity
    HD_NOINLINE void dbl()
    {
        if (is_inf()) return;
        F U = Y.dbl();
        F V = U.sqr();
        F W = U * V;
        F S = X * V;
        F M = X.sqr();
        M = M.dbl() + M;
        F X3 = M.sqr() - S - S;
        Y = M * (S - X3) - W * Y;
        X = X3;
        ZZ = ZZ * V;
        ZZZ = ZZZ * W;
    }

    // *this += p2.  12M + 2S.
    HD_NOINLINE void add(const xyzz_t& p2)
    {
        if (p2.is_inf()) return;
        if (is_inf()) { *this = p2; return; }
        F U1 = X * p2.ZZ;
        F S1 = Y * p2.ZZZ;
        F P = p2.X * ZZ - U1;
        F R = p2.Y * ZZZ - S1;
        if (P.is_zero()) {
            if (R.is_zero()) dbl();
            else set_inf();
            return;
        }
        F PP = P.sqr();
        F PPP = P * PP;
        F Q = U1 * PP;
        F X3 = R.sqr() - PPP - Q - Q;
        Y = R * (Q - X3) - S1 * PPP;
        X = X3;
        ZZ = ZZ * p2.ZZ * PP;
        ZZZ = ZZZ * p2.ZZZ * PPP;
    }


    // ---- variants for the bucket-reduction kernels: the same formulae with every product going
    // through the shared copies of the Montgomery ladder (F::mul_shared / sqr_shared / msub_shared)
    // and the point routine itself inlined, exactly like madd().  The plain add()/dbl() above
    // inline fourteen ladders (~100 KB of code): fine for cold code, but the running-sum kernels
    // then stall on instruction fetch (they ran at 40 % of the accumulate kernel's per-product rate).
    HD void dbl_hot()
    {
        if (is_inf()) return;
        F U = Y.dbl();
        F V = F::sqr_shared(U);
        F W = F::mul_shared(U, V);
        F S = F::mul_shared(X, V);
        F M = F::sqr_shared(X);
        M = M.dbl() + M;
        F X3 = F::sqr_shared(M) - S - S;
        Y = F::msub_shared(M, S - X3, W, Y);
        X = X3;
        ZZ = F::mul_shared(ZZ, V);
        ZZZ = F::mul_shared(ZZZ, W);
    }
    HD void add_hot(const xyzz_t& p2)
    {
        if (p2.is_inf()) return;
        if (is_inf()) { *this = p2; return; }
        F U1 = F::mul_shared(X, p2.ZZ);
        F S1 = F::mul_shared(Y, p2.ZZZ);
        F P = F::mul_shared(p2.X, ZZ) - U1;
        F R = F::mul_shared(p2.Y, ZZZ) - S1;
        if (P.is_zero()) {
            if (R.is_zero()) dbl_hot();
            else set_inf();
            return;
        }
        F PP = F::sqr_shared(P);
        F PPP = F::mul_shared(P, PP);
        F Q = F::mul_shared(U1, PP);
        F X3 = F::sqr_shared(R) - PPP - Q - Q;
        Y = F::msub_shared(R, Q - X3, S1, PPP);
        X = X3;
        ZZ = F::mul_shared(F::mul_shared(ZZ, p2.ZZ), PP);
        ZZZ = F::mul_shared(F::mul_shared(ZZZ, p2.ZZZ), PPP);
    }

    // (X*ZZ, Y*ZZZ, ZZ): Z := ZZ  (ec/xyzz_t.hpp:87-90)
    HD jacobian_t<F> to_jacobian() const
    {
        jacobian_t<F> r;
        if (is_inf()) { r.X = F::zero(); r.Y = F::zero(); r.Z = F::zero(); return r; }
        r.X = X * ZZ;
        r.Y = Y * ZZZ;
        r.Z = ZZ;
        return r;
    }
};

}  // namespace ec
