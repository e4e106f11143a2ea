// Pre-reduction of the bucket lists by BATCHED AFFINE additions (one level).
//
// The accumulate kernel spends 10 field multiplications per point (XYZZ mixed add, 8M + 2S).  An
// affine addition costs one inversion plus 3 multiplications, and Montgomery's trick turns many
// independent inversions into 3 multiplications each plus one shared inversion.  The pairs
// (entry 2i, entry 2i+1) of every bucket list are independent, so this stage replaces each
// bucket's list of L points by ceil(L/2) pair sums (an odd last entry is copied), at ~6.7
// multiplications per pair; the accumulate kernel then folds lists of half the length, reading
// the sums sequentially instead of gathering points.  (The reference adds every point in XYZZ
// form, msm/pippenger.cuh:198-207; ff/batch_inversion.hpp is its only batched-inversion code.)
//
//   counts1[t] = ceil(counts[t] / 2)    (0 for heavy buckets: the cooperative kernels own them)
//   off1[t]    = exclusive prefix of counts1 inside window w;  winbase[w] = outputs before window w
//   output o = winbase[w] + off1[t] + i  <->  pair i of slot t
//   forward : thread = K consecutive outputs; denominators d_j, running products pre[j] = d_0..d_j,
//             the thread's total T = pre[K-1]
//   invert  : Tinv = 1/T, M totals per thread (Montgomery's trick again, one Fermat inversion each)
//   backward: 1/d_j = Tinv_run * pre[j-1], Tinv_run *= d_j; lambda, x3, y3 -> out[o] (affine)
// Every body is per-thread and independent of its neighbours (HD: the CPU single-stepper in
// tests/emu/msm_emu.cpp runs the same code).
#pragma once
#include "msm_core.cuh"

namespace msm {

constexpr uint32_t PAIR_K = 16;          // outputs per thread
constexpr uint32_t PAIR_M = 64;          // thread totals per inversion (3 KB of local memory per thread)

struct PairCursor {                      // position of an output in the bucket structure
    uint32_t t, i;                       // slot, pair index inside it
};

// counts1 for every slot (kernel: one thread per slot)
HD void pair_counts_body(const Config& cfg, const uint32_t* counts, uint32_t* counts1, uint32_t t)
{
    const uint32_t c = counts[t];
    counts1[t] = c > cfg.heavy ? 0 : (c + 1) >> 1;
}

// slot holding output `o` (o < winbase[nwins]): the last slot whose first output is <= o
HD PairCursor pair_locate(const Config& cfg, const uint32_t* off1, const uint32_t* winbase, uint32_t o)
{
    uint32_t w = 0;
    while (w + 1 < cfg.nwins && winbase[w + 1] <= o) w++;
    const uint32_t x = o - winbase[w];
    const uint32_t* row = off1 + ((size_t)w << cfg.lg_nb);
    uint32_t lo = 0, hi = (1u << cfg.lg_nb) - 1;          // invariant: row[lo] <= x
    while (lo < hi) {
        uint32_t mid = (lo + hi + 1) >> 1;
        if (row[mid] <= x) lo = mid;
        else hi = mid - 1;
    }
    return PairCursor{(w << cfg.lg_nb) + lo, x - row[lo]};
}

// the two inputs of pair (t, i) and the denominator of their sum
template<class F>
struct PairTerm {
    ec::affine_t<F> p1, p2;
    F d;                                 // never zero
    uint32_t kind;                       // 0 chord, 1 tangent, 2 result = p1, 3 result = p2, 4 result = infinity
};

template<class F>
HD PairTerm<F> pair_term(const Config& cfg, const uint32_t* points, const uint32_t* sorted,
                         const uint32_t* offsets, const uint32_t* counts, PairCursor c)
{
    const uint32_t* run = sorted + (size_t)(c.t >> cfg.lg_nb) * row_stride(cfg) + offsets[c.t];
    PairTerm<F> r;
    r.p1 = load_point<F>(points, run[2 * c.i]);
    r.d = F::one();
    if (2 * c.i + 1 >= counts[c.t]) { r.kind = 2; r.p2 = r.p1; return r; }          // odd tail: copy
    r.p2 = load_point<F>(points, run[2 * c.i + 1]);
    const bool inf1 = r.p1.X.is_zero() && r.p1.Y.is_zero(), inf2 = r.p2.X.is_zero() && r.p2.Y.is_zero();
    if (inf2) { r.kind = inf1 ? 4 : 2; return r; }
    if (inf1) { r.kind = 3; return r; }
    if (r.p1.X == r.p2.X) {
        if (r.p1.Y == r.p2.Y && !r.p1.Y.is_zero()) { r.kind = 1; r.d = r.p1.Y + r.p1.Y; }
        else r.kind = 4;                                                            // P + (-P)
        return r;
    }
    r.kind = 0;
    r.d = r.p2.X - r.p1.X;
    return r;
}

// one coordinate (X: which = 0, Y: which = 1, sign applied) of the point an entry names
template<class F>
HD F load_coord(const uint32_t* points, uint32_t entry, int which)
{
    const uint32_t* p = points + (size_t)(entry & 0x7fffffffu) * 2 * F::N + which * F::N;
    F v;
#if defined(__CUDA_ARCH__)
    static_assert(F::N % 4 == 0, "a coordinate must be a whole number of 16-byte words");
#pragma unroll
    for (int k = 0; k < F::N / 4; k++) {
        uint4 q = __ldg(reinterpret_cast<const uint4*>(p) + k);
        v.l[4 * k] = q.x; v.l[4 * k + 1] = q.y; v.l[4 * k + 2] = q.z; v.l[4 * k + 3] = q.w;
    }
#else
    for (int k = 0; k < F::N; k++) v.l[k] = p[k];
#endif
    if (which && (entry >> 31)) v = v.neg();
    return v;
}

// the denominator alone, from the X coordinates (half the gather traffic of pair_term); Y is
// fetched only for the rare x == 0 and x1 == x2 cases.  Must agree with pair_term bit for bit.
template<class F>
HD F pair_denominator(const Config& cfg, const uint32_t* points, const uint32_t* sorted,
                      const uint32_t* offsets, const uint32_t* counts, PairCursor c)
{
    const uint32_t* run = sorted + (size_t)(c.t >> cfg.lg_nb) * row_stride(cfg) + offsets[c.t];
    if (2 * c.i + 1 >= counts[c.t]) return F::one();
    const uint32_t e1 = run[2 * c.i], e2 = run[2 * c.i + 1];
    const F x1 = load_coord<F>(points, e1, 0), x2 = load_coord<F>(points, e2, 0);
    if (x2.is_zero() && load_coord<F>(points, e2, 1).is_zero()) return F::one();
    if (x1.is_zero() && load_coord<F>(points, e1, 1).is_zero()) return F::one();
    if (x1 == x2) {
        const F y1 = load_coord<F>(points, e1, 1), y2 = load_coord<F>(points, e2, 1);
        if (y1 == y2 && !y1.is_zero()) return y1 + y1;
        return F::one();
    }
    return x2 - x1;
}

template<class F> HD void pair_store_f(uint32_t* dst, const F& v)
{
#pragma unroll
    for (int k = 0; k < F::N; k++) dst[k] = v.l[k];
}
template<class F> HD F pair_load_f(const uint32_t* src)
{
    F v;
#pragma unroll
    for (int k = 0; k < F::N; k++) v.l[k] = src[k];
    return v;
}

// walk to the next output: next pair of the slot, or the first pair of the next non-empty slot
HD void pair_advance(const uint32_t* counts1, PairCursor& c)
{
    if (++c.i < counts1[c.t]) return;
    c.i = 0;
    do { c.t++; } while (counts1[c.t] == 0);              // the caller stops before the last output
}

// forward pass of thread `tid` over outputs [o0 + tid*K, ...): pre is laid out [j][thread]
// (coalesced), `nthreads` threads in this launch, `total` = winbase[nwins] outputs exist
template<class F>
HD void pair_forward_body(const Config& cfg, const uint32_t* points, const uint32_t* sorted,
                          const uint32_t* offsets, const uint32_t* counts, const uint32_t* counts1,
                          const uint32_t* off1, const uint32_t* winbase, uint32_t o0, uint32_t nthreads,
                          uint32_t* pre, uint32_t* totals, uint32_t tid)
{
    const uint32_t total = winbase[cfg.nwins];
    const uint32_t first = o0 + tid * PAIR_K;
    F acc = F::one();
    if (first < total) {
        PairCursor c = pair_locate(cfg, off1, winbase, first);
        for (uint32_t j = 0; j < PAIR_K && first + j < total; j++) {
            acc = F::mul_shared(acc, pair_denominator<F>(cfg, points, sorted, offsets, counts, c));
            pair_store_f<F>(pre + ((size_t)j * nthreads + tid) * F::N, acc);
            if (first + j + 1 < total) pair_advance(counts1, c);
        }
    }
    pair_store_f<F>(totals + (size_t)tid * F::N, acc);
}

// totals[0..n) -> their inverses, PAIR_M per thread
template<class F>
HD void pair_invert_body(uint32_t* totals, uint32_t n, uint32_t tid)
{
    const uint32_t first = tid * PAIR_M;
    if (first >= n) return;
    const uint32_t m = n - first < PAIR_M ? n - first : PAIR_M;
    F run[PAIR_M];
    F acc = F::one();
    for (uint32_t j = 0; j < m; j++) {
        acc = F::mul_shared(acc, pair_load_f<F>(totals + (size_t)(first + j) * F::N));
        run[j] = acc;
    }
    F inv = acc.inv();
    for (uint32_t j = m; j-- > 0;) {
        F v = pair_load_f<F>(totals + (size_t)(first + j) * F::N);
        pair_store_f<F>(totals + (size_t)(first + j) * F::N, j ? F::mul_shared(inv, run[j - 1]) : inv);
        inv = F::mul_shared(inv, v);
    }
}

// backward pass: the thread's outputs in reverse order
template<class F>
HD void pair_backward_body(const Config& cfg, const uint32_t* points, const uint32_t* sorted,
                           const uint32_t* offsets, const uint32_t* counts, const uint32_t* counts1,
                           const uint32_t* off1, const uint32_t* winbase, uint32_t o0, uint32_t nthreads,
                           const uint32_t* pre, const uint32_t* totals_inv, uint32_t* out, uint32_t tid)
{
    const uint32_t total = winbase[cfg.nwins];
    const uint32_t first = o0 + tid * PAIR_K;
    if (first >= total) return;
    const uint32_t cnt = total - first < PAIR_K ? total - first : PAIR_K;
    PairCursor cur[PAIR_K];
    cur[0] = pair_locate(cfg, off1, winbase, first);
    for (uint32_t j = 1; j < cnt; j++) { cur[j] = cur[j - 1]; pair_advance(counts1, cur[j]); }
    F inv = pair_load_f<F>(totals_inv + (size_t)tid * F::N);
    constexpr int W = 2 * F::N;
    for (uint32_t j = cnt; j-- > 0;) {
        PairTerm<F> term = pair_term<F>(cfg, points, sorted, offsets, counts, cur[j]);
        F dinv = j ? F::mul_shared(inv, pair_load_f<F>(pre + ((size_t)(j - 1) * nthreads + tid) * F::N)) : inv;
        inv = F::mul_shared(inv, term.d);
        ec::affine_t<F> r;
        if (term.kind <= 1) {
            F num;
            if (term.kind == 0) num = term.p2.Y - term.p1.Y;
            else { F xx = F::mul_shared(term.p1.X, term.p1.X); num = xx + xx + xx; }
            const F lambda = F::mul_shared(num, dinv);
            r.X = F::mul_shared(lambda, lambda) - term.p1.X - term.p2.X;
            r.Y = F::mul_shared(lambda, term.p1.X - r.X) - term.p1.Y;
        } else if (term.kind == 2) {
            r = term.p1;
        } else if (term.kind == 3) {
            r = term.p2;
        } else {
            r.X = F::zero(); r.Y = F::zero();
        }
        uint32_t* dst = out + (size_t)(first + j) * W;
        pair_store_f<F>(dst, r.X);
        pair_store_f<F>(dst + F::N, r.Y);
    }
}

}  // namespace msm
