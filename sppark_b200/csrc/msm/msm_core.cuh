// Pippenger bucket MSM: per-thread bodies of every kernel on the path, written HD so that
// tests/emu/msm_emu.cpp can single-step the same logic on the CPU.
//
// Pipeline (one slice of points, all device-resident):
//   count      scalars -> signed c-bit digits, histogram per (window, bucket)   [L2 atomics]
//   scan       per-window exclusive prefix -> bucket offsets, list of heavy buckets
//   scatter    scalars -> digits again, point index (+sign) into its bucket's slot
//   accumulate every lane owns one bucket at a time and streams its points through an XYZZ
//              mixed add; lanes fetch the next bucket from a global counter the moment they
//              finish, so a warp never waits for its longest bucket
//   heavy      buckets longer than `heavy` entries: one CTA each, strided partial sums + tree
//   reduce     sum_b (b+1)*B[w][b] by chunked running sums, then radix-G combine levels
//   finish     Horner over the windows, XYZZ -> Jacobian
//
// Reference counterparts: breakdown (msm/pippenger.cuh:72-121), sort (msm/sort.cuh:366),
// accumulate (:145-223), batch_addition (msm/batch_addition.cuh:134), integrate (:225-296),
// host collect (:627-727).  Digit convention differs (plain two's-complement-free signed
// windows here, Booth there); only the group element is part of the contract
// (poc/msm-cuda/tests/msm.rs:27-38 compares after affine normalisation).
#pragma once
#include <algorithm>
#include "../ec/xyzz.cuh"

namespace msm {

struct Config {
    uint32_t wbits;        // c: window width
    uint32_t nwins;        // ceil(256 / c)
    uint32_t lg_nb;        // c - 1: log2(buckets per window)
    uint32_t npoints;
    uint32_t heavy;        // buckets with more entries go to the cooperative kernel
    uint32_t heavy_chunk;  // entries of a heavy bucket folded by one CTA
    uint32_t merge;        // 0: first slice of points (buckets start empty); 1: add into the buckets
};

HD uint32_t atomic_inc(uint32_t* p, uint32_t v = 1)
{
#if defined(__CUDA_ARCH__)
    return atomicAdd(p, v);
#else
    uint32_t old = *p;
    *p += v;
    return old;
#endif
}

// 256-bit little-endian scalar -> signed digits d_w in (-2^(c-1), 2^(c-1)], sum d_w 2^(cw) = s.
struct Digits {
    uint32_t s[8];
    uint32_t carry;
    HD explicit Digits(const uint32_t* p) : carry(0)
    {
#if defined(__CUDA_ARCH__)
        uint4 a = reinterpret_cast<const uint4*>(p)[0], b = reinterpret_cast<const uint4*>(p)[1];
        s[0] = a.x; s[1] = a.y; s[2] = a.z; s[3] = a.w;
        s[4] = b.x; s[5] = b.y; s[6] = b.z; s[7] = b.w;
#else
        for (int i = 0; i < 8; i++) s[i] = p[i];
#endif
        // Bit 255 is ignored, as the reference ignores every bit from `nbits` up
        // (msm/pippenger.cuh:33-70, nbits = 255 or less for all supported scalar fields): with it
        // cleared the top window can never carry out, also when the window width divides 256, so
        // un-reduced inputs give a deterministic result instead of one that depends on npoints.
        s[7] &= 0x7fffffffu;
    }
    // windows must be requested in order w = 0, 1, ...; returns bucket (|d|-1) and sign,
    // or false for a zero digit
    HD bool next(uint32_t w, uint32_t c, uint32_t& bucket, uint32_t& neg)
    {
        uint32_t off = w * c, i = off >> 5, sh = off & 31;
        uint32_t lo = i < 8 ? s[i] : 0, hi = i + 1 < 8 ? s[i + 1] : 0;
        uint32_t raw = sh ? (lo >> sh) | (hi << (32 - sh)) : lo;
        raw = (c < 32 ? raw & ((1u << c) - 1) : raw) + carry;
        const uint32_t half = 1u << (c - 1);
        if (raw > half) {
            neg = 1;
            carry = 1;
            raw = (1u << c) - raw;             // magnitude of the negative digit
        } else {
            neg = 0;
            carry = 0;
        }
        bucket = raw - 1;
        return raw != 0;
    }
};

// ---- count / scatter -----------------------------------------------------------------
HD void count_body(const Config& cfg, const uint32_t* scalars, uint32_t* counts, uint32_t i)
{
    Digits d(scalars + 8 * (size_t)i);
    for (uint32_t w = 0; w < cfg.nwins; w++) {
        uint32_t b, neg;
        if (d.next(w, cfg.wbits, b, neg))
            atomic_inc(&counts[((size_t)w << cfg.lg_nb) + b]);
    }
}

// windows [w0, w1) only: digits below w0 are still walked for their carry
HD void scatter_body(const Config& cfg, const uint32_t* scalars, uint32_t* cursor,
                     uint32_t* sorted, uint32_t i, uint32_t w0, uint32_t w1)
{
    Digits d(scalars + 8 * (size_t)i);
    for (uint32_t w = 0; w < w1; w++) {
        uint32_t b, neg;
        if (d.next(w, cfg.wbits, b, neg) && w >= w0) {
            uint32_t pos = atomic_inc(&cursor[((size_t)w << cfg.lg_nb) + b]);
            sorted[(size_t)w * cfg.npoints + pos] = i | (neg << 31);
        }
    }
}

// ---- point gather -----------------------------------------------------------------------
template<class F>
HD ec::affine_t<F> load_point(const uint32_t* points, uint32_t entry)
{
    constexpr int W = 2 * F::N;                       // words per affine point
    const uint32_t* p = points + (size_t)(entry & 0x7fffffffu) * W;
    ec::affine_t<F> a;
#if defined(__CUDA_ARCH__)
    static_assert(W % 4 == 0, "affine point must be a whole number of 16-byte words");
    uint32_t buf[W];
#pragma unroll
    for (int k = 0; k < W / 4; k++) {
        uint4 v = __ldg(reinterpret_cast<const uint4*>(p) + k);
        buf[4 * k] = v.x; buf[4 * k + 1] = v.y; buf[4 * k + 2] = v.z; buf[4 * k + 3] = v.w;
    }
#pragma unroll
    for (int k = 0; k < F::N; k++) { a.X.l[k] = buf[k]; a.Y.l[k] = buf[F::N + k]; }
#else
    for (int k = 0; k < F::N; k++) { a.X.l[k] = p[k]; a.Y.l[k] = p[F::N + k]; }
#endif
    if (entry >> 31) a.Y = a.Y.neg();
    return a;
}

template<class F>
HD void store_bucket(uint32_t* buckets, size_t slot, const ec::xyzz_t<F>& b)
{
    constexpr int W = 4 * F::N;
    uint32_t* p = buckets + slot * W;
#pragma unroll
    for (int k = 0; k < F::N; k++) {
        p[k] = b.X.l[k]; p[F::N + k] = b.Y.l[k]; p[2 * F::N + k] = b.ZZZ.l[k]; p[3 * F::N + k] = b.ZZ.l[k];
    }
}

template<class F>
HD ec::xyzz_t<F> load_bucket(const uint32_t* buckets, size_t slot)
{
    constexpr int W = 4 * F::N;
    const uint32_t* p = buckets + slot * W;
    ec::xyzz_t<F> b;
#pragma unroll
    for (int k = 0; k < F::N; k++) {
        b.X.l[k] = p[k]; b.Y.l[k] = p[F::N + k]; b.ZZZ.l[k] = p[2 * F::N + k]; b.ZZ.l[k] = p[3 * F::N + k];
    }
    return b;
}

// ---- accumulate: one lane, many buckets ---------------------------------------------------
// Every lane repeatedly claims the next (window,bucket) from `task_counter` and folds that
// bucket's points.  Empty buckets are written as infinity, heavy ones are skipped (the
// cooperative kernel owns them).
// Direct mode (DIRECT = true; msm_pair.cuh): the lists were pre-reduced to pair sums stored
// consecutively in `points`, slot t owning counts1[t] of them from winbase[w] + off1[t] on; `sorted`
// is not read.
template<class F, bool DIRECT = false>
HD void accumulate_body(const Config& cfg, const uint32_t* points, const uint32_t* sorted,
                        const uint32_t* offsets, const uint32_t* counts, uint32_t* buckets,
                        uint32_t* task_counter, const uint32_t* counts1 = nullptr,
                        const uint32_t* off1 = nullptr, const uint32_t* winbase = nullptr)
{
    const uint32_t total = cfg.nwins << cfg.lg_nb;
    ec::xyzz_t<F> acc;
    const uint32_t* run = nullptr;
    uint32_t t = 0, k = 0, cnt = 0, direct_base = 0;
    bool open = false, live = true;
    // ONE loop, one mixed add per trip, the whole warp in lock step: a lane that finishes its
    // bucket swaps in the next one on the spot and re-joins the warp for the very next add.
    // (A nested "for each bucket / for each point" loop idles every lane until the longest
    // bucket of the warp is done: 26 of 32 lanes active in the round-1 profile.)  The vote at
    // the top is also the reconvergence point after the divergent bucket switch.
    for (;;) {
        if (live && k == cnt) {
            if (open) store_bucket<F>(buckets, t, acc);
            open = false;
            for (;;) {
                t = atomic_inc(task_counter);
                if (t >= total) { live = false; break; }
                t = total - 1 - t;          // top window first: its few, long buckets must not be the tail
                cnt = counts[t];
                if (cnt == 0) {
                    if (!cfg.merge) {
                        acc.set_inf();
                        store_bucket<F>(buckets, t, acc);
                    }
                    continue;
                }
                if (cnt > cfg.heavy) continue;
                break;
            }
            if (DIRECT && live) {
                cnt = counts1[t];
                direct_base = winbase[t >> cfg.lg_nb] + off1[t];
            }
            if (live) {
                if (!DIRECT) run = sorted + (size_t)(t >> cfg.lg_nb) * cfg.npoints + offsets[t];
                if (cfg.merge) acc = load_bucket<F>(buckets, t);
                else acc.set_inf();
                k = 0;
                open = true;
            }
        }
#if defined(__CUDA_ARCH__)
        if (!__any_sync(0xffffffffu, live)) return;
#else
        if (!live) return;
#endif
        if (live) acc.madd(load_point<F>(points, DIRECT ? direct_base + k++ : run[k++]));
        // (an explicit prefetch.global.L2 of the next point was tried: no gain on the GPU the
        //  kernel was first tuned on -- the resident warps per SM already cover the gather latency)
    }
}

// ---- reduce: chunked running sums -----------------------------------------------------------
// level 1: item = one bucket.  Thread (w, chunk) folds L = 2^lg_l consecutive buckets into
//   S = sum B_k,  R = sum (k+1) B_k   (k local)
template<class F>
HD void reduce1_body(const Config& cfg, const uint32_t* buckets, uint32_t lg_l,
                     uint32_t* outR, uint32_t* outS, uint32_t item)
{
    const size_t first = (size_t)item << lg_l;
    ec::xyzz_t<F> acc, res;
    acc.set_inf();
    res.set_inf();
    for (uint32_t k = 1u << lg_l; k-- > 0;) {
        acc.add_hot(load_bucket<F>(buckets, first + k));
        res.add_hot(acc);
    }
    store_bucket<F>(outR, item, res);
    store_bucket<F>(outS, item, acc);
}

// level >= 2: G consecutive items (R_i, S_i), each spanning 2^lg_span buckets, become one:
//   S = sum S_i,  R = sum R_i + 2^lg_span * sum i*S_i
template<class F>
HD void combine_body(const uint32_t* inR, const uint32_t* inS, uint32_t G, uint32_t lg_span,
                     uint32_t* outR, uint32_t* outS, uint32_t item)
{
    const size_t first = (size_t)item * G;
    ec::xyzz_t<F> acc, weighted, rsum;
    acc.set_inf();
    weighted.set_inf();
    rsum.set_inf();
    for (uint32_t i = G; i-- > 0;) {
        rsum.add_hot(load_bucket<F>(inR, first + i));
        acc.add_hot(load_bucket<F>(inS, first + i));
        if (i) weighted.add_hot(acc);                    // sum_{i>=1} i*S_i
    }
    for (uint32_t d = 0; d < lg_span; d++) weighted.dbl_hot();
    rsum.add_hot(weighted);
    store_bucket<F>(outR, item, rsum);
    store_bucket<F>(outS, item, acc);
}

// finish: out = sum_w 2^(c*w) * R_w, as a Jacobian point with canonical coordinates
template<class F>
HD void finish_body(const Config& cfg, const uint32_t* winR, uint32_t* out_jacobian)
{
    ec::xyzz_t<F> acc = load_bucket<F>(winR, cfg.nwins - 1);
    for (uint32_t w = cfg.nwins - 1; w-- > 0;) {
        for (uint32_t d = 0; d < cfg.wbits; d++) acc.dbl_hot();
        acc.add_hot(load_bucket<F>(winR, w));
    }
    ec::jacobian_t<F> j = acc.to_jacobian();
#pragma unroll
    for (int k = 0; k < F::N; k++) {
        out_jacobian[k] = j.X.l[k]; out_jacobian[F::N + k] = j.Y.l[k]; out_jacobian[2 * F::N + k] = j.Z.l[k];
    }
}

// window width minimising the measured cost model (fitted on an earlier GPU; not refitted for H100):
//   per (point, window): 1 mixed add + ~0.11 for count/scatter;  per bucket: ~5.5 mixed-add
//   equivalents for the two full adds of the running sum
inline uint32_t choose_wbits(size_t npoints)
{
    uint32_t best = 4;
    double best_cost = 1e300;
    for (uint32_t c = 4; c <= 22; c++) {
        uint32_t nwins = (256 + c - 1) / c;
        double cost = (double)nwins * (1.11 * (double)npoints + 5.5 * (double)(1u << (c - 1)));
        // a top window of only a few bits puts npoints / 2^e entries into each of its 2^e buckets: the
        // count / scatter atomics collide on them and they go through the heavy-bucket path; at 2^23
        // points c = 16 (no thin window) measured faster than the c = 18 this model ranks first
        // without the term (on the GPU the model was fitted on).  Left alone below 2^22 points,
        // where the table was tuned without it.
        const uint32_t e = 256 - (nwins - 1) * c;                 // bits of the top window
        if (npoints >= ((size_t)1 << 22) && e <= 10 && (npoints >> e) > 2048) cost += 1.25 * (double)npoints;
        if (cost < best_cost) { best_cost = cost; best = c; }
    }
    if (const char* env = getenv("SPPARK_B200_MSM_WBITS")) {
        uint32_t c = (uint32_t)atoi(env);
        if (c >= 3 && c <= 24) best = c;                 // >= 4 buckets per window (scan_kernel loads uint4)
    }
    return best;
}

inline Config make_config(size_t npoints)
{
    Config cfg;
    cfg.wbits = choose_wbits(npoints);
    cfg.nwins = (256 + cfg.wbits - 1) / cfg.wbits;
    cfg.lg_nb = cfg.wbits - 1;
    cfg.npoints = (uint32_t)npoints;
    // a bucket is "heavy" when one lane folding it alone would take longer than that lane's fair
    // share of the whole job (57k lanes: the resident lane count the constant was chosen for; an
    // H100 keeps ~51k resident, close enough for a threshold): such buckets are cut into chunks
    // and spread over CTAs.  At 2^26 points the share is ~15k entries (nothing is heavy for uniform
    // scalars, the long top-window buckets are simply queued first); at 2^16 it is ~25, and the
    // three 16k-entry buckets of the top window must not be left to three single lanes.
    const uint64_t share = (uint64_t)cfg.nwins * npoints / 57000;
    cfg.heavy = (uint32_t)std::min<uint64_t>(std::max<uint64_t>(share, 256), 16384);
    cfg.heavy_chunk = std::min<uint32_t>(std::max<uint32_t>(4 * cfg.heavy, 2048), 16384);
    cfg.merge = 0;
    if (const char* env = getenv("SPPARK_B200_MSM_HEAVY")) cfg.heavy = (uint32_t)atoi(env);
    return cfg;
}

}  // namespace msm
