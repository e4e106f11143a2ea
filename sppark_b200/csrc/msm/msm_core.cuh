// Pippenger bucket MSM: per-thread bodies of every kernel on the path, written HD so that
// tests/emu/msm_emu.cpp (the pipeline) and tests/emu/msm_sort_emu.cpp (the bin sort) can
// single-step the same logic on the CPU.
//
// Pipeline (one slice of points, all device-resident):
//   sort       scalars -> signed c-bit digits -> (window, bucket) lists of point index (+sign),
//              bucket counts and offsets, list of heavy buckets; two passes over coarse bins
//              (bin histogram + partition, then one CTA per bin), see "sort" below
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

// Precomputed tables (copies > 1): the points are stored K times, copy k holding 2^(c*V*k) * P_i at
// row i + k * copy_stride.  Digit w = k*V + v of scalar i then goes to bucket set v with the point
// of copy k, so V = ceil(D / K) bucket sets and V - 1 Horner steps cover all D digits.  With one
// copy the digit count D and the bucket-set count are both nwins; everything below loops over
// the bucket sets ("windows") as before.
//
// Batches (nvecs = G > 1): G scalar vectors against the same points, one after the other in the scalar
// array (vector g's scalars start g * npoints * swords words after vector 0).  Each vector has its own
// V = nwins / G bucket sets: set s belongs to vector s / V, and vector g's digit w goes to set
// g V + digit_slot(w).  The bucket entry stays point | sign << 31, since the points are shared, and the
// kernels after the sort see nwins sets as for one vector.
struct Config {
    uint32_t wbits;        // c: window width
    uint32_t nwins;        // bucket sets G V; per vector V: D = ceil((nbits + 1) / c) without a table, ceil(D / K) with one
    uint32_t lg_nb;        // c - 1: log2(buckets per window)
    uint32_t npoints;
    uint32_t heavy;        // buckets with more entries go to the cooperative kernel
    uint32_t heavy_chunk;  // entries of a heavy bucket folded by one CTA
    uint32_t merge;        // 0: first slice of points (buckets start empty); 1: add into the buckets
    uint32_t copies;       // K: copies of the points in the table (1: plain points)
    uint32_t copy_stride;  // points between two copies: the table's point count, not the slice's
    // the scalar format: scalar i is the little-endian integer in words [i * swords, (i + 1) * swords),
    // bits from nbits up are ignored (255 and 8 words for the 32-byte entries).  Two 16-bit fields fill
    // the struct's padding, so the kernel parameters after a Config keep their offsets.
    uint16_t nbits;        // 1 .. min(255, 32 * swords)
    uint16_t swords;       // 32-bit words per scalar: 1, 2, 4 or 8
    uint32_t nvecs;        // G: scalar vectors of the group (1 without a batch)
};

// V: the bucket sets of one vector
HD uint32_t vec_sets(const Config& cfg) { return cfg.nvecs == 1 ? cfg.nwins : cfg.nwins / cfg.nvecs; }
// the geometry of G vectors, each with the sets of the one-vector geometry cfg
inline Config group_config(Config cfg, uint32_t nvecs)
{
    cfg.nwins *= nvecs;
    cfg.nvecs = nvecs;
    return cfg;
}

// digits per scalar, D = ceil((nbits + 1) / c) (equal to nwins without a table): the top digit never
// carries out of the last window; ceil(256 / c) for 255-bit scalars
HD uint32_t digits_for(uint32_t nbits, uint32_t wbits) { return (nbits + wbits) / wbits; }
HD uint32_t digit_count(const Config& cfg) { return digits_for(cfg.nbits, cfg.wbits); }
// entries per bucket-set row of `staging` / `sorted`: every copy of every point of the slice
// (a 32-bit product: a table keeps copies * points < 2^31, the bucket entry's index range)
HD size_t row_stride(const Config& cfg) { return cfg.copies * cfg.npoints; }

// digit w of point i -> bucket set v = w mod V of its vector (returned) and entry
// (i + (w / V) * copy_stride) | sign << 31
HD uint32_t digit_slot(const Config& cfg, uint32_t w, uint32_t i, uint32_t neg, uint32_t& entry)
{
    if (cfg.copies == 1) { entry = i | (neg << 31); return w; }
    const uint32_t V = vec_sets(cfg), k = w / V;
    entry = (i + k * cfg.copy_stride) | (neg << 31);
    return w - k * V;
}

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

// little-endian scalar of SW 32-bit words -> signed digits d_w in (-2^(c-1), 2^(c-1)], sum d_w 2^(cw) = s.
// The scalar is read with one load of its width (32, 64 or 128 bits; two 128-bit loads for 8 words).
template<uint32_t SW>
struct Digits {
    uint32_t s[SW];
    uint32_t carry;
    HD Digits(const uint32_t* p, uint32_t nbits) : carry(0)
    {
#if defined(__CUDA_ARCH__)
        if constexpr (SW == 1) {
            s[0] = *p;
        } else if constexpr (SW == 2) {
            const uint2 a = *reinterpret_cast<const uint2*>(p);
            s[0] = a.x; s[1] = a.y;
        } else {
#pragma unroll
            for (uint32_t k = 0; k < SW / 4; k++) {
                const uint4 a = reinterpret_cast<const uint4*>(p)[k];
                s[4 * k] = a.x; s[4 * k + 1] = a.y; s[4 * k + 2] = a.z; s[4 * k + 3] = a.w;
            }
        }
#else
        for (uint32_t k = 0; k < SW; k++) s[k] = p[k];
#endif
        // Bits from nbits up are ignored, as the reference ignores every bit from its `nbits` up
        // (msm/pippenger.cuh:33-70; 255 for the 32-byte entries): with them cleared the top window
        // can never carry out, also when the window width divides nbits + 1, so un-reduced inputs
        // give a deterministic result instead of one that depends on npoints.
#pragma unroll
        for (uint32_t k = 0; k < SW; k++) {
            if (32 * k >= nbits) s[k] = 0;
            else if (nbits - 32 * k < 32) s[k] &= (1u << (nbits - 32 * k)) - 1;
        }
    }
    // windows must be requested in order w = 0, 1, ...; returns bucket (|d|-1) and sign,
    // or false for a zero digit
    HD bool next(uint32_t w, uint32_t c, uint32_t& bucket, uint32_t& neg)
    {
        uint32_t off = w * c, i = off >> 5, sh = off & 31;
        uint32_t lo = i < SW ? s[i] : 0, hi = i + 1 < SW ? s[i + 1] : 0;
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

// first scalar word of vector g
HD size_t vec_offset(const Config& cfg, uint32_t g) { return (size_t)g * cfg.npoints * cfg.swords; }

// fn(Digits<swords>&) for scalar i of vector g of a scalar array in the format of cfg (host-side bodies:
// the device kernels are instantiated per width instead)
template<class Fn>
HD void with_digits(const Config& cfg, const uint32_t* scalars, uint32_t i, Fn fn, uint32_t g = 0)
{
    scalars += vec_offset(cfg, g);
    switch (cfg.swords) {
    case 1: { Digits<1> d(scalars + (size_t)i, cfg.nbits); fn(d); break; }
    case 2: { Digits<2> d(scalars + 2 * (size_t)i, cfg.nbits); fn(d); break; }
    case 4: { Digits<4> d(scalars + 4 * (size_t)i, cfg.nbits); fn(d); break; }
    default: { Digits<8> d(scalars + 8 * (size_t)i, cfg.nbits); fn(d); break; }
    }
}

// ---- direct sort: one counter and one cursor per (window, bucket) ----------------------------
// The plain form of the sort below: count every entry into its bucket, exclusive prefix per window,
// place every entry at its bucket's cursor.  It produces the same counts, offsets and bucket lists
// (up to the order inside a bucket), and the CPU single-stepper of the whole pipeline
// (tests/emu/msm_emu.cpp) runs it.  The device does not: with 2^(c-1) buckets per window its
// random 4-byte stores keep more partly written lines open than L2 holds.
// g: the vector of a batch (Config::nvecs) whose scalar i is counted / placed
HD void count_body(const Config& cfg, const uint32_t* scalars, uint32_t* counts, uint32_t i, uint32_t g = 0)
{
    const uint32_t s0 = g * vec_sets(cfg);
    with_digits(cfg, scalars, i, [&](auto& d) {
        const uint32_t nd = digit_count(cfg);
        for (uint32_t w = 0; w < nd; w++) {
            uint32_t b, neg, entry;
            if (d.next(w, cfg.wbits, b, neg))
                atomic_inc(&counts[((size_t)(s0 + digit_slot(cfg, w, i, neg, entry)) << cfg.lg_nb) + b]);
        }
    }, g);
}

// digits [w0, w1) only: digits below w0 are still walked for their carry
HD void scatter_body(const Config& cfg, const uint32_t* scalars, uint32_t* cursor,
                     uint32_t* sorted, uint32_t i, uint32_t w0, uint32_t w1, uint32_t g = 0)
{
    const uint32_t s0 = g * vec_sets(cfg);
    with_digits(cfg, scalars, i, [&](auto& d) {
        for (uint32_t w = 0; w < w1; w++) {
            uint32_t b, neg, entry;
            if (d.next(w, cfg.wbits, b, neg) && w >= w0) {
                const uint32_t v = s0 + digit_slot(cfg, w, i, neg, entry);
                uint32_t pos = atomic_inc(&cursor[((size_t)v << cfg.lg_nb) + b]);
                sorted[(size_t)v * row_stride(cfg) + pos] = entry;
            }
        }
    }, g);
}

// ---- sort: (window, bucket) lists of point indices -----------------------------------------
// Two passes over coarse bins, so that no phase writes to more places at once than L2 holds:
//   bin histogram  bin = (w << lg_bins) + (bucket >> s_w): 2^lg_bins bins per window
//   partition      every (point, window) entry appended at its bin's cursor in `staging`
//                  (index | sign << 31, bucket): the open write frontier is one line per bin
//   bin sort       one CTA per bin: histogram of its 2^s_w buckets in shared memory, counts /
//                  offsets / heavy buckets, entries placed through shared memory, written out whole
//   overflow       bins over the CTA's capacity: the same three steps with global atomics
// Bin b of window w occupies the same range [w*n + bin_base, + bin_count) in `staging` and in
// `sorted`, since its buckets are consecutive.
constexpr uint32_t SORT_SMAX = 12;      // a bin spans at most 2^12 buckets (its shared histogram)
constexpr uint32_t SORT_LG_FILL = 13;   // bins hold about 2^13 entries of a uniform window

// bits of the top window's digit magnitude: bits from nbits up are ignored, so the window holds bits
// (W-1)c..nbits-1 plus the carry and its buckets are < 2^(nbits - (W-1)c) (at most 2^(c-1); 2^0 when
// c divides nbits and the window holds only the carry)
HD uint32_t top_window_bits(const Config& cfg)
{
    const uint32_t e = cfg.nbits - (vec_sets(cfg) - 1) * cfg.wbits;
    return e < cfg.lg_nb ? e : cfg.lg_nb;
}
// with a table the thin top digit shares its bucket set with full-width digits: every set is full.
// v: the set's index inside its vector (w mod V for set w)
HD uint32_t window_bits(const Config& cfg, uint32_t v)
{   return v + 1 < vec_sets(cfg) || cfg.copies > 1 ? cfg.lg_nb : top_window_bits(cfg);   }
// buckets per bin of a window with vector-local index v: 2^s_v, so the window's used buckets [0, 2^ub)
// make <= 2^lg_bins bins
HD uint32_t bin_shift(const Config& cfg, uint32_t lg_bins, uint32_t v)
{
    const uint32_t ub = window_bits(cfg, v);
    return ub > lg_bins ? ub - lg_bins : 0;
}

// bins per window for a slice of n points: about 2^SORT_LG_FILL entries per bin, at most 2^SORT_SMAX
// buckets per bin, at least 4 bins (the bin scan reads them four at a time), at most 2^15 (the bin
// histogram keeps one window's counters in shared memory); past 2^28 points bins grow instead
inline uint32_t sort_lg_bins(const Config& cfg, size_t n)
{
    int lg_n = 0;
    while (((size_t)1 << lg_n) < n) lg_n++;
    int lb = std::max(std::min(lg_n - (int)SORT_LG_FILL, 15), (int)cfg.lg_nb - (int)SORT_SMAX);
    lb = std::min(lb, (int)cfg.lg_nb);
    return (uint32_t)std::max(lb, 2);
}

// bucket range [b0, b0 + nbk) of bin `bin` (window-local) of window w; false for a bin past the
// window's used buckets (always empty)
HD bool bin_buckets(const Config& cfg, uint32_t lg_bins, uint32_t w, uint32_t bin, uint32_t& b0, uint32_t& nbk)
{
    const uint32_t v = w % vec_sets(cfg), s = bin_shift(cfg, lg_bins, v), ub = window_bits(cfg, v);
    b0 = bin << s;
    nbk = 1u << s;
    return b0 < (1u << ub);
}

// the last used bin of a window also owns the offsets of the never-used buckets above it
HD bool last_bin(const Config& cfg, uint32_t lg_bins, uint32_t w, uint32_t bin)
{
    const uint32_t v = w % vec_sets(cfg);
    return ((bin + 1) << bin_shift(cfg, lg_bins, v)) == (1u << window_bits(cfg, v));
}

// every digit of point i of vector g in order: fn(set, nonzero, bin (global), bucket, entry), with set
// g V + v and entry from digit_slot (without a table and batch: set = digit index, entry = i | sign << 31).
// Digits >= w_end are not visited.  `valid` false: fn sees only zero digits (the tail lanes of a warp
// that must still take part in its collective operations).  SW: cfg.swords, the scalar width the
// kernel is built for.
template<uint32_t SW = 8, class Fn>
HD void for_each_digit(const Config& cfg, uint32_t lg_bins, const uint32_t* scalars, uint32_t i, bool valid,
                       uint32_t w_end, Fn fn, uint32_t g = 0)
{
    Digits<SW> d(scalars + (size_t)g * cfg.npoints * SW + SW * (size_t)(valid ? i : 0), cfg.nbits);
    const uint32_t V = vec_sets(cfg), s0 = g * V;
    // bin_shift of the vector's top set and of the others, once per scalar
    const uint32_t top = bin_shift(cfg, lg_bins, V - 1), full = bin_shift(cfg, lg_bins, 0);
    for (uint32_t w = 0; w < w_end; w++) {
        uint32_t b, neg, entry;
        const bool nz = d.next(w, cfg.wbits, b, neg) && valid;
        const uint32_t v = digit_slot(cfg, w, i, neg, entry), s = s0 + v;
        fn(s, nz, (s << lg_bins) + (nz ? b >> (v + 1 < V ? full : top) : 0), b, entry);
    }
}

// heavy bucket h: heavy_list[3h] = slot, [3h+1] = first chunk, [3h+2] = #chunks; chunk_map[c] = h
HD void register_heavy(const Config& cfg, uint32_t t, uint32_t cnt, uint32_t* ctrl, uint32_t* heavy_list,
                       uint32_t* chunk_map)
{
    if (cnt <= cfg.heavy) return;
    const uint32_t h = atomic_inc(&ctrl[1]), nch = (cnt + cfg.heavy_chunk - 1) / cfg.heavy_chunk;
    const uint32_t first_chunk = atomic_inc(&ctrl[2], nch);
    heavy_list[3 * h] = t;
    heavy_list[3 * h + 1] = first_chunk;
    heavy_list[3 * h + 2] = nch;
    for (uint32_t q = 0; q < nch; q++) chunk_map[first_chunk + q] = h;
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
                if (!DIRECT) run = sorted + (size_t)(t >> cfg.lg_nb) * row_stride(cfg) + offsets[t];
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

// finish: out = sum_w 2^(c*w) * R_w over the V bucket sets of one vector, as a Jacobian point with
// canonical coordinates (with a table, set v holds every digit v + kV, its factor 2^(cVk) already in
// the points).  winR: the vector's first set; a batch's vector g reads from set g V on.
template<class F>
HD void finish_body(const Config& cfg, const uint32_t* winR, uint32_t* out_jacobian)
{
    const uint32_t V = vec_sets(cfg);
    ec::xyzz_t<F> acc = load_bucket<F>(winR, V - 1);
    for (uint32_t w = V - 1; w-- > 0;) {
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
// over the W = ceil((nbits + 1) / c) windows of nbits-bit scalars (255: the 32-byte entries)
inline uint32_t choose_wbits(size_t npoints, uint32_t nbits)
{
    uint32_t best = 4;
    double best_cost = 1e300;
    for (uint32_t c = 4; c <= 22; c++) {
        uint32_t nwins = digits_for(nbits, c);
        double cost = (double)nwins * (1.11 * (double)npoints + 5.5 * (double)(1u << (c - 1)));
        // a top window of only a few bits puts npoints / 2^e entries into each of its 2^e buckets: the
        // count / scatter atomics collide on them and they go through the heavy-bucket path; at 2^23
        // points c = 16 (no thin window) measured faster than the c = 18 this model ranks first
        // without the term (on the GPU the model was fitted on).  Left alone below 2^22 points,
        // where the table was tuned without it.
        const uint32_t e = nbits + 1 - (nwins - 1) * c;           // bits of the top window
        if (npoints >= ((size_t)1 << 22) && e <= 10 && (npoints >> e) > 2048) cost += 1.25 * (double)npoints;
        if (cost < best_cost) { best_cost = cost; best = c; }
    }
    if (const char* env = getenv("SPPARK_B200_MSM_WBITS")) {
        uint32_t c = (uint32_t)atoi(env);
        if (c >= 3 && c <= 24) best = c;                 // >= 4 buckets per window (pair_scan_kernel loads uint4)
    }
    return best;
}
inline uint32_t choose_wbits(size_t npoints) { return choose_wbits(npoints, 255); }

// a bucket is "heavy" when one lane folding it alone would take longer than that lane's fair
// share of the whole job (57k lanes: the resident lane count the constant was chosen for; an
// H100 keeps ~51k resident, close enough for a threshold): such buckets are cut into chunks
// and spread over CTAs.  At 2^26 points the share is ~15k entries (nothing is heavy for uniform
// scalars, the long top-window buckets are simply queued first); at 2^16 it is ~25, and the
// three 16k-entry buckets of the top window must not be left to three single lanes.
// `entries`: (point, digit) entries of the whole job, D * npoints.
inline void set_heavy(Config& cfg, uint64_t entries)
{
    const uint64_t share = entries / 57000;
    cfg.heavy = (uint32_t)std::min<uint64_t>(std::max<uint64_t>(share, 256), 16384);
    cfg.heavy_chunk = std::min<uint32_t>(std::max<uint32_t>(4 * cfg.heavy, 2048), 16384);
    if (const char* env = getenv("SPPARK_B200_MSM_HEAVY")) cfg.heavy = (uint32_t)atoi(env);
}

// the geometry of an MSM over npoints scalars of scalar_bytes bytes whose bits from nbits up are ignored
inline Config make_config(size_t npoints, uint32_t nbits, uint32_t scalar_bytes)
{
    Config cfg;
    cfg.wbits = choose_wbits(npoints, nbits);
    cfg.nwins = digits_for(nbits, cfg.wbits);
    cfg.lg_nb = cfg.wbits - 1;
    cfg.npoints = (uint32_t)npoints;
    cfg.merge = 0;
    cfg.copies = 1;
    cfg.copy_stride = (uint32_t)npoints;
    cfg.nbits = (uint16_t)nbits;
    cfg.swords = (uint16_t)(scalar_bytes / 4);
    cfg.nvecs = 1;
    set_heavy(cfg, (uint64_t)cfg.nwins * npoints);
    return cfg;
}
inline Config make_config(size_t npoints) { return make_config(npoints, 255, 32); }

// ---- precomputed tables ---------------------------------------------------------------------
// The geometry of a table of width c built for at most `copies` copies: V = ceil(D / K) bucket sets,
// K_used = ceil(D / V) <= K copies stored (more would add no set), for an MSM over n points of a
// table whose copies are `stride` points apart.  The heavy threshold follows the D * n entries.
// With nbits-bit scalars only the digits w < D_b = ceil((nbits + 1) / c) are walked: the sets stay
// the table's V and copies 0 .. ceil(D_b / V) - 1 are read; when D_b <= V only copy 0 is, and the
// geometry is the plain one of width c (D_b sets, its thin top window included).
inline Config config_for_table(size_t n, uint32_t wbits, uint32_t copies, size_t stride, uint32_t nbits,
                               uint32_t scalar_bytes)
{
    Config cfg;
    const uint32_t D = digits_for(255, wbits), K = std::max(1u, std::min(copies, D)), V = (D + K - 1) / K;
    const uint32_t Db = digits_for(nbits, wbits);
    cfg.wbits = wbits;
    cfg.nwins = std::min(V, Db);
    cfg.lg_nb = wbits - 1;
    cfg.npoints = (uint32_t)n;
    cfg.merge = 0;
    cfg.copies = (Db + cfg.nwins - 1) / cfg.nwins;
    cfg.copy_stride = (uint32_t)stride;
    cfg.nbits = (uint16_t)nbits;
    cfg.swords = (uint16_t)(scalar_bytes / 4);
    cfg.nvecs = 1;
    set_heavy(cfg, (uint64_t)Db * n);
    return cfg;
}
inline Config config_for_table(size_t n, uint32_t wbits, uint32_t copies, size_t stride)
{   return config_for_table(n, wbits, copies, stride, 255, 32);   }

// N points, at most K copies: make_config for K = 1; otherwise the width c in [4, 24] minimising the
// window cost model of choose_wbits re-scored for the table, 1.11 D N + 5.5 V 2^(c-1) (the mixed
// adds stay D N, the bucket work is paid once per set).  SPPARK_B200_MSM_WBITS overrides c.
inline Config make_config_precomputed(size_t npoints, uint32_t copies)
{
    if (copies <= 1) return make_config(npoints);
    uint32_t best = 4;
    double best_cost = 1e300;
    for (uint32_t c = 4; c <= 24; c++) {
        const uint32_t D = digits_for(255, c), V = (D + copies - 1) / copies;
        const double cost = 1.11 * (double)D * (double)npoints + 5.5 * (double)V * (double)(1u << (c - 1));
        if (cost < best_cost) { best_cost = cost; best = c; }
    }
    if (const char* env = getenv("SPPARK_B200_MSM_WBITS")) {
        uint32_t c = (uint32_t)atoi(env);
        if (c >= 3 && c <= 24) best = c;
    }
    return config_for_table(npoints, best, copies, npoints);
}

}  // namespace msm
