// msm_t<Curve>: device-side Pippenger driver (the role of the reference's msm_t,
// msm/pippenger.cuh:325-747).  Kernels are thin __global__ wrappers over msm_core.cuh.
#pragma once
#include "../util/gpu.cuh"
#include "msm_core.cuh"
#include "msm_pair.cuh"

namespace msm {

#ifndef SPPARK_B200_ACC_THREADS
# define SPPARK_B200_ACC_THREADS 128
#endif
#ifndef SPPARK_B200_ACC_MIN_BLOCKS
# define SPPARK_B200_ACC_MIN_BLOCKS 3
#endif
constexpr uint32_t ACC_THREADS = SPPARK_B200_ACC_THREADS;       // accumulate CTA size
constexpr uint32_t HEAVY_THREADS = 128;

static __global__ void count_kernel(const Config cfg, const uint32_t* scalars, uint32_t* counts)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < cfg.npoints; i += gridDim.x * blockDim.x)
        count_body(cfg, scalars, counts, i);
}


// control block: [0] task counter, [1] #heavy buckets, [2] #chunks
// heavy bucket h: heavy_list[3h] = slot, [3h+1] = first chunk, [3h+2] = #chunks; chunk_map[c] = h
// one CTA (1024 threads) per window: exclusive prefix of the bucket histogram in tiles of 4096
// counters (one 128-bit load per thread, warp-shuffle scans); heavy buckets get chunked
static __global__ void __launch_bounds__(1024)
scan_kernel(const Config cfg, const uint32_t* counts, uint32_t* offsets, uint32_t* cursor,
            uint32_t* ctrl, uint32_t* heavy_list, uint32_t* chunk_map)
{
    __shared__ uint32_t warp_tot[32];
    const uint32_t w = blockIdx.x, nb = 1u << cfg.lg_nb;            // nb >= 8: a multiple of 4
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const size_t base = (size_t)w << cfg.lg_nb;
    uint32_t carry = 0;                                             // total of the tiles before this one
    for (uint32_t t0 = 0; t0 < nb; t0 += 4096) {
        const uint32_t b = t0 + threadIdx.x * 4;
        uint4 c = make_uint4(0, 0, 0, 0);
        if (b < nb) c = *reinterpret_cast<const uint4*>(counts + base + b);
        const uint32_t s = c.x + c.y + c.z + c.w;
        uint32_t x = s;                                             // inclusive scan inside the warp
#pragma unroll
        for (uint32_t d = 1; d < 32; d <<= 1) {
            uint32_t y = __shfl_up_sync(0xffffffffu, x, d);
            if (lane >= d) x += y;
        }
        if (lane == 31) warp_tot[wid] = x;
        __syncthreads();
        if (wid == 0) {
            uint32_t t = warp_tot[lane];
#pragma unroll
            for (uint32_t d = 1; d < 32; d <<= 1) {
                uint32_t y = __shfl_up_sync(0xffffffffu, t, d);
                if (lane >= d) t += y;
            }
            warp_tot[lane] = t;
        }
        __syncthreads();
        uint4 r;
        r.x = carry + (wid ? warp_tot[wid - 1] : 0) + x - s;
        r.y = r.x + c.x;
        r.z = r.y + c.y;
        r.w = r.z + c.z;
        carry += warp_tot[31];
        if (b < nb) {
            *reinterpret_cast<uint4*>(offsets + base + b) = r;
            *reinterpret_cast<uint4*>(cursor + base + b) = r;
            const uint32_t cc[4] = {c.x, c.y, c.z, c.w};
#pragma unroll
            for (uint32_t k = 0; k < 4; k++) {
                if (cc[k] > cfg.heavy) {
                    uint32_t h = atomicAdd(&ctrl[1], 1), nch = (cc[k] + cfg.heavy_chunk - 1) / cfg.heavy_chunk;
                    uint32_t first_chunk = atomicAdd(&ctrl[2], nch);
                    heavy_list[3 * h] = (uint32_t)(base + b + k);
                    heavy_list[3 * h + 1] = first_chunk;
                    heavy_list[3 * h + 2] = nch;
                    for (uint32_t q = 0; q < nch; q++) chunk_map[first_chunk + q] = h;
                }
            }
        }
        __syncthreads();                                            // warp_tot is reused by the next tile
    }
}

static __global__ void scatter_kernel(const Config cfg, const uint32_t* scalars, uint32_t* cursor, uint32_t* sorted,
                                      uint32_t w0, uint32_t w1)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < cfg.npoints; i += gridDim.x * blockDim.x)
        scatter_body(cfg, scalars, cursor, sorted, i, w0, w1);
}

// ---- batched-affine pre-reduction of the bucket lists (msm_pair.cuh) ---------------------------
static __global__ void pair_counts_kernel(const Config cfg, const uint32_t* counts, uint32_t* counts1, uint32_t nslots)
{
    for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < nslots; t += gridDim.x * blockDim.x)
        pair_counts_body(cfg, counts, counts1, t);
}

// one CTA (1024 threads) per window: window-local exclusive prefix of counts1, window total
static __global__ void __launch_bounds__(1024)
pair_scan_kernel(const Config cfg, const uint32_t* counts1, uint32_t* off1, uint32_t* wintotal)
{
    __shared__ uint32_t warp_tot[32];
    const uint32_t w = blockIdx.x, nb = 1u << cfg.lg_nb, lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const size_t base = (size_t)w << cfg.lg_nb;
    uint32_t carry = 0;
    for (uint32_t t0 = 0; t0 < nb; t0 += 4096) {
        const uint32_t b = t0 + threadIdx.x * 4;
        uint4 c = make_uint4(0, 0, 0, 0);
        if (b < nb) c = *reinterpret_cast<const uint4*>(counts1 + base + b);
        const uint32_t s = c.x + c.y + c.z + c.w;
        uint32_t x = s;
#pragma unroll
        for (uint32_t d = 1; d < 32; d <<= 1) {
            uint32_t y = __shfl_up_sync(0xffffffffu, x, d);
            if (lane >= d) x += y;
        }
        if (lane == 31) warp_tot[wid] = x;
        __syncthreads();
        if (wid == 0) {
            uint32_t t = warp_tot[lane];
#pragma unroll
            for (uint32_t d = 1; d < 32; d <<= 1) {
                uint32_t y = __shfl_up_sync(0xffffffffu, t, d);
                if (lane >= d) t += y;
            }
            warp_tot[lane] = t;
        }
        __syncthreads();
        uint4 r;
        r.x = carry + (wid ? warp_tot[wid - 1] : 0) + x - s;
        r.y = r.x + c.x;
        r.z = r.y + c.y;
        r.w = r.z + c.z;
        carry += warp_tot[31];
        if (b < nb) *reinterpret_cast<uint4*>(off1 + base + b) = r;
        __syncthreads();
    }
    if (threadIdx.x == 0) wintotal[w] = carry;
}

static __global__ void pair_winbase_kernel(const Config cfg, const uint32_t* wintotal, uint32_t* winbase)
{
    if (blockIdx.x || threadIdx.x) return;
    uint32_t run = 0;
    for (uint32_t w = 0; w < cfg.nwins; w++) { winbase[w] = run; run += wintotal[w]; }
    winbase[cfg.nwins] = run;
}

template<class F>
__global__ void __launch_bounds__(128)
pair_forward_kernel(const Config cfg, const uint32_t* points, const uint32_t* sorted, const uint32_t* offsets,
                    const uint32_t* counts, const uint32_t* counts1, const uint32_t* off1, const uint32_t* winbase,
                    uint32_t o0, uint32_t nthreads, uint32_t* pre, uint32_t* totals)
{
    const uint32_t tid = blockIdx.x * blockDim.x + threadIdx.x;
    if (tid < nthreads)
        pair_forward_body<F>(cfg, points, sorted, offsets, counts, counts1, off1, winbase, o0, nthreads, pre, totals, tid);
}

template<class F>
__global__ void __launch_bounds__(128)
pair_invert_kernel(uint32_t* totals, uint32_t n)
{
    pair_invert_body<F>(totals, n, blockIdx.x * blockDim.x + threadIdx.x);
}

template<class F>
__global__ void __launch_bounds__(128)
pair_backward_kernel(const Config cfg, const uint32_t* points, const uint32_t* sorted, const uint32_t* offsets,
                     const uint32_t* counts, const uint32_t* counts1, const uint32_t* off1, const uint32_t* winbase,
                     uint32_t o0, uint32_t nthreads, const uint32_t* pre, const uint32_t* totals_inv, uint32_t* out)
{
    const uint32_t tid = blockIdx.x * blockDim.x + threadIdx.x;
    if (tid < nthreads)
        pair_backward_body<F>(cfg, points, sorted, offsets, counts, counts1, off1, winbase, o0, nthreads, pre,
                              totals_inv, out, tid);
}

template<class F>
__global__ void __launch_bounds__(ACC_THREADS, (F::N > 12 ? 2 : SPPARK_B200_ACC_MIN_BLOCKS))
accumulate_direct_kernel(const Config cfg, const uint32_t* sums, const uint32_t* offsets, const uint32_t* counts,
                         uint32_t* buckets, uint32_t* task_counter, const uint32_t* counts1, const uint32_t* off1,
                         const uint32_t* winbase)
{
    accumulate_body<F, true>(cfg, sums, nullptr, offsets, counts, buckets, task_counter, counts1, off1, winbase);
}

template<class F>
__global__ void __launch_bounds__(ACC_THREADS, (F::N > 12 ? 2 : SPPARK_B200_ACC_MIN_BLOCKS))
accumulate_kernel(const Config cfg, const uint32_t* points, const uint32_t* sorted,
                  const uint32_t* offsets, const uint32_t* counts, uint32_t* buckets,
                  uint32_t* task_counter)
{
    accumulate_body<F>(cfg, points, sorted, offsets, counts, buckets, task_counter);
}

// block-wide sum of one xyzz per thread through shared memory; result valid in thread 0
template<class F>
DEV void block_sum(ec::xyzz_t<F>& acc, uint32_t* tree)
{
    store_bucket<F>(tree, threadIdx.x, acc);
    __syncthreads();
    for (uint32_t d = blockDim.x / 2; d > 0; d >>= 1) {
        if (threadIdx.x < d) {
            acc.add_hot(load_bucket<F>(tree, threadIdx.x + d));
            store_bucket<F>(tree, threadIdx.x, acc);
        }
        __syncthreads();
    }
}

// heavy buckets, phase A: one CTA per cfg.heavy_chunk entries -> one partial sum per chunk, so a
// bucket holding most of the points is spread over the whole GPU
template<class F>
__global__ void __launch_bounds__(HEAVY_THREADS)
heavy_chunks_kernel(const Config cfg, const uint32_t* points, const uint32_t* sorted,
                    const uint32_t* offsets, const uint32_t* counts, const uint32_t* ctrl,
                    const uint32_t* heavy_list, const uint32_t* chunk_map, uint32_t* partials)
{
    extern __shared__ __align__(16) uint32_t tree[];         // HEAVY_THREADS xyzz slots
    const uint32_t nchunks = ctrl[2];
    for (uint32_t ch = blockIdx.x; ch < nchunks; ch += gridDim.x) {
        const uint32_t h = chunk_map[ch], t = heavy_list[3 * h], k0 = (ch - heavy_list[3 * h + 1]) * cfg.heavy_chunk;
        const uint32_t cnt = counts[t], k1 = min(k0 + cfg.heavy_chunk, cnt);
        const uint32_t* run = sorted + (size_t)(t >> cfg.lg_nb) * cfg.npoints + offsets[t];
        ec::xyzz_t<F> acc;
        acc.set_inf();
        for (uint32_t k = k0 + threadIdx.x; k < k1; k += blockDim.x)
            acc.madd(load_point<F>(points, run[k]));
        block_sum<F>(acc, tree);
        if (threadIdx.x == 0) store_bucket<F>(partials, ch, acc);
        __syncthreads();
    }
}

// phase B: one CTA per heavy bucket folds that bucket's chunk partials
template<class F>
__global__ void __launch_bounds__(HEAVY_THREADS)
heavy_fold_kernel(const Config cfg, const uint32_t* ctrl, const uint32_t* heavy_list,
                  const uint32_t* partials, uint32_t* buckets)
{
    extern __shared__ __align__(16) uint32_t tree[];
    const uint32_t nheavy = ctrl[1];
    for (uint32_t h = blockIdx.x; h < nheavy; h += gridDim.x) {
        const uint32_t t = heavy_list[3 * h], first = heavy_list[3 * h + 1], nch = heavy_list[3 * h + 2];
        ec::xyzz_t<F> acc;
        acc.set_inf();
        for (uint32_t k = threadIdx.x; k < nch; k += blockDim.x)
            acc.add_hot(load_bucket<F>(partials, first + k));
        block_sum<F>(acc, tree);
        if (threadIdx.x == 0) {
            if (cfg.merge) acc.add_hot(load_bucket<F>(buckets, t));
            store_bucket<F>(buckets, t, acc);
        }
        __syncthreads();
    }
}

// 3 CTAs/SM: the <= 4096 items per window of a 2^26 MSM (416 CTAs) then fit one wave of 444
// resident CTAs; at 255 registers (2 CTAs/SM) they took two
template<class F>
__global__ void __launch_bounds__(128, (F::N > 12 ? 2 : 3))
reduce1_kernel(const Config cfg, const uint32_t* buckets, uint32_t lg_l, uint32_t nitems,
               uint32_t* outR, uint32_t* outS)
{
    uint32_t item = blockIdx.x * blockDim.x + threadIdx.x;
    if (item < nitems) reduce1_body<F>(cfg, buckets, lg_l, outR, outS, item);
}

template<class F>
__global__ void __launch_bounds__(128)
combine_kernel(const uint32_t* inR, const uint32_t* inS, uint32_t G, uint32_t lg_span,
               uint32_t nitems, uint32_t* outR, uint32_t* outS)
{
    uint32_t item = blockIdx.x * blockDim.x + threadIdx.x;
    if (item < nitems) combine_body<F>(inR, inS, G, lg_span, outR, outS, item);
}

template<class F>
__global__ void finish_kernel(const Config cfg, const uint32_t* winR, uint32_t* out)
{
    if (blockIdx.x == 0 && threadIdx.x == 0) finish_body<F>(cfg, winR, out);
}

// ---- finish on four lanes -------------------------------------------------------------------------
// The Horner combination of the window sums is one dependent chain of nwins*c doublings; what can
// run side by side are the multiplications INSIDE a point operation: a doubling (dbl-2008-s-1) is
// three rounds of independent products {V = U^2, Q = X^2}, {W = UV, S = XV, M^2}, {M(S-X3), WY,
// ZZ*V, ZZZ*W}, a full addition four.  Lanes 0..3 of one warp execute the shared ladder in
// lock-step on different operands (one instruction stream, SIMD), values travel through a few
// shared-memory slots: 3 ladder latencies per doubling instead of 9, 4 per addition instead of
// 14 (the same group element as finish_body, which the CPU single-stepper keeps running).
template<class F> struct Par4 {
    enum { sX, sY, sZZZ, sZZ, sA, sB, sC, sD, sE, sF, sG, sH, NS };
    // slot i of the accumulator: its four coordinates first, then eight scratch values that
    // several accumulators of one lane group may share
    struct Slots {
        F* pt;
        F* tmp;
        __device__ F& operator[](uint32_t i) const { return i < 4 ? pt[i] : tmp[i - 4]; }
    };
    Slots s;
    uint32_t lane;
    unsigned mask;                                          // the four lanes of this group
    __device__ Par4(F* pt, F* tmp, uint32_t lane_, unsigned mask_ = 0xFu) : s{pt, tmp}, lane(lane_), mask(mask_) {}
    __device__ void sync() const { __syncwarp(mask); }
    __device__ ec::xyzz_t<F> get() const
    {
        ec::xyzz_t<F> p;
        p.X = s[sX]; p.Y = s[sY]; p.ZZZ = s[sZZZ]; p.ZZ = s[sZZ];
        return p;
    }
    __device__ void set_inf()
    {
        if (lane == 0) { s[sX] = F::zero(); s[sY] = F::zero(); s[sZZZ] = F::zero(); s[sZZ] = F::zero(); }
        sync();
    }
    __device__ bool is_inf() const { return s[sZZZ].is_zero() && s[sZZ].is_zero(); }

    // lane-wise choice of an operand: every lane then makes THE SAME call of the shared ladder (one
    // instruction stream for the four products; a branch per lane would serialise them)
    __device__ F pick(const F& a0, const F& a1, const F& a2, const F& a3) const
    {
        F r;
#pragma unroll
        for (int i = 0; i < F::N; i++)
            r.l[i] = lane == 0 ? a0.l[i] : lane == 1 ? a1.l[i] : lane == 2 ? a2.l[i] : a3.l[i];
        return r;
    }
    __device__ void put(uint32_t i0, uint32_t i1, uint32_t i2, uint32_t i3, const F& r)
    {   s[lane == 0 ? i0 : lane == 1 ? i1 : lane == 2 ? i2 : i3] = r;   }

    __device__ void dbl()
    {
        if (is_inf()) return;                               // same decision on all four lanes
        const F U = s[sY].dbl(), X = s[sX];
        F r = F::mul_shared(pick(U, X, X, X), pick(U, X, X, X));
        put(sA, sB, sB, sB, r);                             // sA = V = U^2, sB = Q = X^2
        sync();
        const F V = s[sA];
        F M = s[sB];
        M = M.dbl() + M;
        r = F::mul_shared(pick(U, X, M, M), pick(V, V, M, M));
        put(sC, sD, sE, sE, r);                             // sC = W, sD = S, sE = M^2
        sync();
        const F W = s[sC], S = s[sD];
        const F X3 = s[sE] - S - S;
        const F Y = s[sY], ZZ = s[sZZ], ZZZ = s[sZZZ];
        sync();                                             // everyone has read the old point
        r = F::mul_shared(pick(M, W, ZZ, ZZZ), pick(S - X3, Y, V, W));
        put(sF, sG, sZZ, sZZZ, r);
        sync();
        if (lane == 0) { s[sY] = s[sF] - s[sG]; s[sX] = X3; }
        sync();
    }

    // point += p2 (both XYZZ); p2 in registers of every lane
    __device__ void add(const ec::xyzz_t<F>& p2)
    {
        if (p2.is_inf()) return;
        if (is_inf()) {
            if (lane == 0) { s[sX] = p2.X; s[sY] = p2.Y; s[sZZZ] = p2.ZZZ; s[sZZ] = p2.ZZ; }
            sync();
            return;
        }
        const F X1 = s[sX], Y1 = s[sY], ZZZ1 = s[sZZZ], ZZ1 = s[sZZ];
        F r = F::mul_shared(pick(X1, Y1, p2.X, p2.Y), pick(p2.ZZ, p2.ZZZ, ZZ1, ZZZ1));
        put(sA, sB, sC, sD, r);                             // sA = U1, sB = S1, sC = U2, sD = S2
        sync();
        const F U1 = s[sA], S1 = s[sB];
        const F P = s[sC] - U1, R = s[sD] - S1;
        sync();
        if (P.is_zero()) {                                  // same decision on all four lanes
            if (R.is_zero()) dbl();
            else { if (lane == 0) { s[sZZZ] = F::zero(); s[sZZ] = F::zero(); } sync(); }
            return;
        }
        r = F::mul_shared(pick(P, R, ZZ1, ZZZ1), pick(P, R, p2.ZZ, p2.ZZZ));
        put(sE, sF, sG, sH, r);                             // sE = PP, sF = RR, sG = ZZ1*ZZ2, sH = ZZZ1*ZZZ2
        sync();
        const F PP = s[sE], G = s[sG];
        r = F::mul_shared(pick(P, U1, G, G), PP);
        put(sA, sC, sZZ, sZZ, r);                           // sA = PPP, sC = Q, ZZ3
        sync();
        const F PPP = s[sA], Q = s[sC], H = s[sH];
        const F X3 = s[sF] - PPP - Q - Q;
        r = F::mul_shared(pick(R, S1, H, H), pick(Q - X3, PPP, PPP, PPP));
        put(sD, sE, sZZZ, sZZZ, r);                         // T1, T2, ZZZ3
        sync();
        if (lane == 0) { s[sY] = s[sD] - s[sE]; s[sX] = X3; }
        sync();
    }
};

// combine level (see combine_body) with four lanes per item: the chains of a level are G x 3 full
// additions long and there are only a few thousand items, so latency, not throughput, sets its
// time; the additions run as four rounds of lane-parallel products
// four-lane groups per CTA: 20 field elements of shared memory each (30 KB for 48-byte Fp at 32
// groups; Fp2 elements are twice as wide, so half as many groups)
template<class F> struct par_groups { static constexpr uint32_t value = F::N <= 12 ? 32 : 16; };

template<class F>
__global__ void __launch_bounds__(4 * par_groups<F>::value)
combine_par_kernel(const uint32_t* inR, const uint32_t* inS, uint32_t G, uint32_t lg_span,
                   uint32_t nitems, uint32_t* outR, uint32_t* outS)
{
    __shared__ F sm[par_groups<F>::value][20];                   // per group: acc, weighted, rsum, 8 scratch
    const uint32_t grp = threadIdx.x >> 2, lane = threadIdx.x & 3;
    const uint32_t item = blockIdx.x * par_groups<F>::value + grp;
    if (item >= nitems) return;                             // whole groups leave together
    const unsigned mask = 0xFu << ((threadIdx.x & 31) & ~3u);
    F* base = sm[grp];
    Par4<F> acc(base, base + 12, lane, mask), weighted(base + 4, base + 12, lane, mask), rsum(base + 8, base + 12, lane, mask);
    acc.set_inf();
    weighted.set_inf();
    rsum.set_inf();
    const size_t first = (size_t)item * G;
    for (uint32_t i = G; i-- > 0;) {
        rsum.add(load_bucket<F>(inR, first + i));
        acc.add(load_bucket<F>(inS, first + i));
        if (i) weighted.add(acc.get());                     // sum_{i>=1} i*S_i
    }
    for (uint32_t d = 0; d < lg_span; d++) weighted.dbl();
    rsum.add(weighted.get());
    if (lane == 0) {
        store_bucket<F>(outR, item, rsum.get());
        store_bucket<F>(outS, item, acc.get());
    }
}

template<class F>
__global__ void __launch_bounds__(32)
finish_par_kernel(const Config cfg, const uint32_t* winR, uint32_t* out_jacobian)
{
    __shared__ F slots[Par4<F>::NS];
    if (threadIdx.x >= 4) return;
    Par4<F> p(slots, slots + 4, threadIdx.x);
    {
        const ec::xyzz_t<F> top = load_bucket<F>(winR, cfg.nwins - 1);
        if (p.lane == 0) { slots[Par4<F>::sX] = top.X; slots[Par4<F>::sY] = top.Y; slots[Par4<F>::sZZZ] = top.ZZZ; slots[Par4<F>::sZZ] = top.ZZ; }
        p.sync();
    }
    for (uint32_t w = cfg.nwins - 1; w-- > 0;) {
        for (uint32_t d = 0; d < cfg.wbits; d++) p.dbl();
        p.add(load_bucket<F>(winR, w));
    }
    // XYZZ -> Jacobian (X*ZZ, Y*ZZZ, ZZ), canonical limbs; infinity -> all zero
    const bool inf = p.is_inf();
    const F ZZ = slots[Par4<F>::sZZ];
    const F Yf = slots[Par4<F>::sY], ZZZf = slots[Par4<F>::sZZZ];
    const F r = F::mul_shared(p.pick(slots[Par4<F>::sX], Yf, Yf, Yf), p.pick(ZZ, ZZZf, ZZZf, ZZZf));
    if (p.lane < 2)
        for (int k = 0; k < F::N; k++) out_jacobian[p.lane * F::N + k] = inf ? 0 : r.l[k];
    if (p.lane == 2)
        for (int k = 0; k < F::N; k++) out_jacobian[2 * F::N + k] = inf ? 0 : ZZ.l[k];
}

// host rows {X, Y, [flag]} at `stride` bytes -> packed {X, Y}; flagged rows become (0,0)
// (reference: Affine_inf_t::mem_t, ec/affine_t.hpp:91-121; stream_t::HtoD pitch copy)
static __global__ void pack_points_kernel(const uint8_t* in, size_t stride, uint32_t words, bool has_flag,
                                   uint32_t* out, uint32_t npoints)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < npoints; i += gridDim.x * blockDim.x) {
        const uint32_t* src = reinterpret_cast<const uint32_t*>(in + (size_t)i * stride);
        bool inf = has_flag && (in[(size_t)i * stride + 4 * words] & 1);
        for (uint32_t k = 0; k < words; k++) out[(size_t)i * words + k] = inf ? 0 : src[k];
    }
}

template<class F>
class msm_t {
    const gpu_t& gpu;
    static constexpr uint32_t PW = 2 * F::N, BW = 4 * F::N, JW = 3 * F::N;   // words per affine/xyzz/jacobian

public:
    explicit msm_t(const gpu_t& g) : gpu(g) {}

    // ---- a transform in flight: buckets persist across slices of points ----------------------
    struct Job {
        Config cfg;                 // window geometry for the WHOLE MSM; npoints = slice capacity
        size_t nslots, slice_cap;
        uint32_t lg_l, items1;
        uint8_t* blob;
        uint32_t *counts, *offsets, *cursor, *ctrl, *heavy_list, *chunk_map, *partials, *sorted, *buckets;
        uint32_t *R[2], *S[2];
        uint32_t slices_done;
        // batched-affine pre-reduction (msm_pair.cuh), off unless SPPARK_B200_MSM_PAIR=1
        bool pair;
        size_t pair_bound;          // most pair sums one slice can produce
        uint32_t pair_threads;      // threads per forward/backward launch (PAIR_K outputs each)
        uint32_t *counts1, *off1, *wintotal, *winbase, *sums, *pre, *totals;
        // the scratch blob (several GB at 2^26) is released on every exit path, also when a CUDA
        // call between begin() and finish() throws
        cudaStream_t owner;
        Job() : blob(nullptr), owner(nullptr) {}
        Job(const Job&) = delete;
        Job& operator=(const Job&) = delete;
        Job(Job&& o) noexcept { memcpy((void*)this, (const void*)&o, sizeof(Job)); o.blob = nullptr; }
        ~Job() { if (blob) (void)cudaFreeAsync(blob, owner); }
    };

    // total_points fixes the window width; slice_cap is the most points one slice() call may carry
    Job begin(size_t total_points, size_t slice_cap, cudaStream_t stream)
    {
        if (total_points >= (1ull << 31))
            throw cuda_error(-(int)cudaErrorInvalidValue, "msm: npoints must be < 2^31");
        Job j;
        j.cfg = make_config(total_points);
        j.cfg.npoints = (uint32_t)slice_cap;
        j.slice_cap = slice_cap;
        j.nslots = (size_t)j.cfg.nwins << j.cfg.lg_nb;
        j.lg_l = j.cfg.lg_nb > 12 ? j.cfg.lg_nb - 12 : 0;          // <= 4096 running-sum items per window
        j.items1 = j.cfg.nwins << (j.cfg.lg_nb - j.lg_l);
        j.slices_done = 0;
        const size_t entries = (size_t)j.cfg.nwins * slice_cap;
        const size_t heavy_cap = entries / (j.cfg.heavy + 1) + 1;   // most heavy buckets possible
        const size_t chunk_cap = entries / j.cfg.heavy_chunk + heavy_cap; // most chunks possible
        size_t off = 0;
        auto take = [&](size_t bytes) { size_t o = off; off += (bytes + 255) & ~(size_t)255; return o; };
        const size_t o_counts = take(j.nslots * 4), o_offsets = take(j.nslots * 4), o_cursor = take(j.nslots * 4);
        const size_t o_ctrl = take(16), o_heavy = take(heavy_cap * 12), o_cmap = take(chunk_cap * 4);
        const size_t o_partials = take(chunk_cap * BW * 4);
        const size_t o_sorted = take(entries * 4);
        const size_t o_buckets = take(j.nslots * BW * 4);
        const size_t o_r0 = take((size_t)j.items1 * BW * 4), o_s0 = take((size_t)j.items1 * BW * 4);
        const size_t o_r1 = take((size_t)j.items1 * BW * 4 / 2 + 4096), o_s1 = take((size_t)j.items1 * BW * 4 / 2 + 4096);
        // experimental, measured once in round 1 (DESIGN.md section 8): halves the bucket lists with
        // batched affine pair sums before the XYZZ accumulation
        const char* pair_env = getenv("SPPARK_B200_MSM_PAIR");
        j.pair = pair_env && atoi(pair_env) != 0 && entries + j.nslots < (1ull << 31);
        j.pair_bound = (entries + std::min<size_t>(entries, j.nslots) + 1) / 2;
        j.pair_threads = (uint32_t)std::min<size_t>((j.pair_bound + PAIR_K - 1) / PAIR_K, (size_t)1 << 21);
        size_t o_c1 = 0, o_o1 = 0, o_wt = 0, o_wb = 0, o_sums = 0, o_pre = 0, o_tot = 0;
        if (j.pair) {
            o_c1 = take(j.nslots * 4); o_o1 = take(j.nslots * 4);
            o_wt = take((j.cfg.nwins + 1) * 4); o_wb = take((j.cfg.nwins + 1) * 4);
            o_sums = take(j.pair_bound * 2 * F::N * 4);
            o_pre = take((size_t)j.pair_threads * PAIR_K * F::N * 4);
            o_tot = take((size_t)j.pair_threads * F::N * 4);
        }
        CUDA_OK(cudaMallocAsync((void**)&j.blob, off, stream));
        j.owner = stream;
        auto U32 = [&](size_t o) { return reinterpret_cast<uint32_t*>(j.blob + o); };
        j.counts = U32(o_counts); j.offsets = U32(o_offsets); j.cursor = U32(o_cursor);
        j.ctrl = U32(o_ctrl); j.heavy_list = U32(o_heavy); j.chunk_map = U32(o_cmap);
        j.partials = U32(o_partials); j.sorted = U32(o_sorted); j.buckets = U32(o_buckets);
        j.R[0] = U32(o_r0); j.S[0] = U32(o_s0); j.R[1] = U32(o_r1); j.S[1] = U32(o_s1);
        j.counts1 = U32(o_c1); j.off1 = U32(o_o1); j.wintotal = U32(o_wt); j.winbase = U32(o_wb);
        j.sums = U32(o_sums); j.pre = U32(o_pre); j.totals = U32(o_tot);
        g_profile.reset();
        return j;
    }

    // fold `n` (<= slice_cap) device-resident points/scalars into the buckets
    void slice(Job& j, const uint32_t* d_points, const uint32_t* d_scalars, size_t n, cudaStream_t stream)
    {
        if (n == 0) return;
        Config cfg = j.cfg;
        cfg.npoints = (uint32_t)n;
        cfg.merge = j.slices_done ? 1 : 0;
        const uint32_t sms = (uint32_t)gpu.sm_count();
        g_profile.mark("sort", stream);
        CUDA_OK(cudaMemsetAsync(j.counts, 0, j.nslots * 4, stream));
        CUDA_OK(cudaMemsetAsync(j.ctrl, 0, 16, stream));
        const uint32_t nblk = (uint32_t)std::min<size_t>((n + 255) / 256, (size_t)sms * 16);
        count_kernel<<<nblk, 256, 0, stream>>>(cfg, d_scalars, j.counts);
        COUNT_LAUNCH();
        scan_kernel<<<cfg.nwins, 1024, 0, stream>>>(cfg, j.counts, j.offsets, j.cursor, j.ctrl, j.heavy_list, j.chunk_map);
        COUNT_LAUNCH();
        // The scatter writes 4 random bytes per (point, window): with all windows in flight the
        // write set (4*n bytes per window) thrashes L2 and every store costs a 32-byte sector
        // read + write-back in DRAM.  One launch per window confines the write set to one window's
        // slots (4*n bytes, resident in the 50 MB L2 of an H100 up to n = 2^23) at the price of
        // re-reading the scalars per window.
        bool per_window = n >= (1u << 18);
        if (const char* env = getenv("SPPARK_B200_MSM_SCATTER")) per_window = atoi(env) != 0;
        if (per_window) {
            for (uint32_t w = 0; w < cfg.nwins; w++) {
                scatter_kernel<<<nblk, 256, 0, stream>>>(cfg, d_scalars, j.cursor, j.sorted, w, w + 1);
                COUNT_LAUNCH();
            }
        } else {
            scatter_kernel<<<nblk, 256, 0, stream>>>(cfg, d_scalars, j.cursor, j.sorted, 0, cfg.nwins);
            COUNT_LAUNCH();
        }
        CUDA_OK(cudaGetLastError());

        g_profile.mark("accumulate", stream);
        int occ = 1;
        CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, accumulate_kernel<F>, ACC_THREADS, 0));
        if (occ < 1) occ = 1;
        size_t want = (j.nslots + ACC_THREADS - 1) / ACC_THREADS;
        uint32_t acc_blocks = (uint32_t)std::min<size_t>(want, (size_t)sms * occ);
        if (j.pair) {
            const uint32_t nslots = (uint32_t)j.nslots;
            pair_counts_kernel<<<sms * 8, 256, 0, stream>>>(cfg, j.counts, j.counts1, nslots);
            pair_scan_kernel<<<cfg.nwins, 1024, 0, stream>>>(cfg, j.counts1, j.off1, j.wintotal);
            pair_winbase_kernel<<<1, 32, 0, stream>>>(cfg, j.wintotal, j.winbase);
            // the host does not know how many pair sums this slice has (winbase[nwins], on the
            // device): launches cover the bound, threads past the real total return at once
            const size_t bound = ((size_t)cfg.nwins * n + std::min<size_t>((size_t)cfg.nwins * n, j.nslots) + 1) / 2;
            const size_t per_launch = (size_t)j.pair_threads * PAIR_K;
            for (size_t o0 = 0; o0 < bound; o0 += per_launch) {
                const uint32_t nth = (uint32_t)std::min<size_t>(j.pair_threads, (bound - o0 + PAIR_K - 1) / PAIR_K);
                pair_forward_kernel<F><<<(nth + 127) / 128, 128, 0, stream>>>(
                    cfg, d_points, j.sorted, j.offsets, j.counts, j.counts1, j.off1, j.winbase, (uint32_t)o0, nth, j.pre, j.totals);
                pair_invert_kernel<F><<<((nth + PAIR_M - 1) / PAIR_M + 127) / 128, 128, 0, stream>>>(j.totals, nth);
                pair_backward_kernel<F><<<(nth + 127) / 128, 128, 0, stream>>>(
                    cfg, d_points, j.sorted, j.offsets, j.counts, j.counts1, j.off1, j.winbase, (uint32_t)o0, nth, j.pre, j.totals, j.sums);
                COUNT_LAUNCH(); COUNT_LAUNCH(); COUNT_LAUNCH();
            }
            CUDA_OK(cudaGetLastError());
            g_profile.mark("accumulate_sums", stream);
            accumulate_direct_kernel<F><<<acc_blocks, ACC_THREADS, 0, stream>>>(cfg, j.sums, j.offsets, j.counts, j.buckets,
                                                                               j.ctrl, j.counts1, j.off1, j.winbase);
        } else {
            accumulate_kernel<F><<<acc_blocks, ACC_THREADS, 0, stream>>>(cfg, d_points, j.sorted, j.offsets, j.counts,
                                                                        j.buckets, j.ctrl);
        }
        COUNT_LAUNCH();
        g_profile.mark("heavy", stream);
        heavy_chunks_kernel<F><<<sms * 4, HEAVY_THREADS, HEAVY_THREADS * BW * 4, stream>>>(
            cfg, d_points, j.sorted, j.offsets, j.counts, j.ctrl, j.heavy_list, j.chunk_map, j.partials);
        COUNT_LAUNCH();
        heavy_fold_kernel<F><<<sms, HEAVY_THREADS, HEAVY_THREADS * BW * 4, stream>>>(cfg, j.ctrl, j.heavy_list,
                                                                                    j.partials, j.buckets);
        COUNT_LAUNCH();
        CUDA_OK(cudaGetLastError());
        if (getenv("SPPARK_B200_MSM_DEBUG")) {
            uint32_t dbg[3];
            CUDA_OK(cudaMemcpyAsync(dbg, j.ctrl, 12, cudaMemcpyDeviceToHost, stream));
            CUDA_OK(cudaStreamSynchronize(stream));
            fprintf(stderr, "[msm] slice %u n=%u wbits=%u nwins=%u heavy_thr=%u tasks_claimed=%u nheavy=%u nchunks=%u acc_blocks=%u\n",
                    j.slices_done, cfg.npoints, cfg.wbits, cfg.nwins, cfg.heavy, dbg[0], dbg[1], dbg[2], acc_blocks);
        }
        j.slices_done++;
    }

    // running sums over the buckets, Horner over the windows -> d_out (JW words), frees the job
    void finish(Job& j, uint32_t* d_out, cudaStream_t stream)
    {
        if (j.slices_done == 0) {
            CUDA_OK(cudaMemsetAsync(d_out, 0, JW * 4, stream));
        } else {
            const Config& cfg = j.cfg;
            g_profile.mark("reduce", stream);
            reduce1_kernel<F><<<(j.items1 + 127) / 128, 128, 0, stream>>>(cfg, j.buckets, j.lg_l, j.items1, j.R[0], j.S[0]);
            COUNT_LAUNCH();
            uint32_t per_win = 1u << (cfg.lg_nb - j.lg_l), lg_span = j.lg_l, cur = 0;
            while (per_win > 1) {
                uint32_t lg_g = 31 - __builtin_clz(per_win);
                if (lg_g > 4) lg_g = 4;                         // radix 16 keeps the serial chains short
                uint32_t G = 1u << lg_g, nitems = cfg.nwins * (per_win >> lg_g);
                constexpr uint32_t PG = par_groups<F>::value;
                combine_par_kernel<F><<<(nitems + PG - 1) / PG, 4 * PG, 0, stream>>>(j.R[cur], j.S[cur], G, lg_span, nitems,
                                                                                     j.R[cur ^ 1], j.S[cur ^ 1]);
                COUNT_LAUNCH();
                per_win >>= lg_g;
                lg_span += lg_g;
                cur ^= 1;
            }
            g_profile.mark("finish", stream);
            finish_par_kernel<F><<<1, 32, 0, stream>>>(cfg, j.R[cur], d_out);
            COUNT_LAUNCH();
            g_profile.mark("end", stream);
            CUDA_OK(cudaGetLastError());
        }
        CUDA_OK(cudaFreeAsync(j.blob, stream));
        j.blob = nullptr;
    }

    // all inputs device-resident: d_points packed affine, d_scalars 8 words each.
    // d_out: JW words of device memory.  Enqueues on `stream`; no synchronisation.
    void invoke_dev(uint32_t* d_out, const uint32_t* d_points, size_t npoints,
                    const uint32_t* d_scalars, cudaStream_t stream)
    {
        if (npoints == 0) {
            CUDA_OK(cudaMemsetAsync(d_out, 0, JW * 4, stream));
            return;
        }
        Job j = begin(npoints, npoints, stream);
        slice(j, d_points, d_scalars, npoints, stream);
        finish(j, d_out, stream);
    }
};

}  // namespace msm
