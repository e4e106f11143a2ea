// Polynomial helpers over the NTT fields: inclusive prefix sum / product, division by (x - z),
// multi-point evaluation, batch inversion.  SURVEY.md section 8 row f4: the reference's
// polynomial/{prefix_op,div_by_x_minus_z,evaluate}.cuh and ff/batch_inversion.hpp.
//
// The reference writes each of these as ONE cooperative kernel with grid-wide barriers between a
// local phase, a cross-block carry phase and an apply phase.  Here:
//  * prefix_op and div_by_x_minus_z are the same tiled scan.  Long inputs: three ordinary launches
//    (tile aggregates, a scan of the aggregates, rescan with carries), no ordering between CTAs;
//    inputs whose tiles are all resident: ONE cooperative launch with a single grid barrier, the
//    tile kept in registers across it; up to two tiles: one plain launch.  Division by (x - z) is the scan of
//    b[i] = c[i] + z * b[i+1]  from the top coefficient down: the carry that crosses k elements
//    is weighted by z^k, and since every level of the hierarchy (thread, lane, warp, tile) spans
//    a fixed number of elements the weights are a handful of constants held in shared memory;
//    the scan of the tile aggregates is the same recurrence with z^TILE in the place of z.
//  * evaluate is a strided Horner (thread g owns coefficients g, g+G, ...: one multiplication per
//    coefficient and point, contiguous reads) followed by  sum_t s_t * x^t  over the CTA by
//    shuffles, one partial per CTA and a one-CTA finish per point.
//  * batch inversion shares ONE field inversion per CTA: prefix and suffix products over the CTA
//    give every thread the inverse of its own chunk product; for long arrays of wide elements the
//    inversions themselves are batched the same way, one level up.
// All arithmetic is on the field's memory format (arith<F> below), the same the NTT entry points
// use, so buffers pass between NTT and these helpers unchanged.
#pragma once
#include "../ff/gl64.cuh"
#include "../ff/bb31.cuh"
#include "../ff/mont_ntt.cuh"
#include "../util/gpu.cuh"
#if defined(__CUDACC__)
# include <cooperative_groups.h>
#endif

namespace poly {

// ---- arithmetic on the memory format -------------------------------------------------------------
// "data" values are what sits in memory; "constants" (z, x and their powers) may live in another
// domain when that saves work: cmul(data, constant) -> data, kmul(constant, constant) -> constant.
template<class F> struct arith {                       // Montgomery fields: one closed domain
    typedef typename F::T T;
    static HD T zero() { T z{}; return z; }
    static HD T one() { return F::one(); }
    static HD T load(const T& a) { return F::load(a); }
    static HD T add(const T& a, const T& b) { return F::add(a, b); }
    static HD T dmul(const T& a, const T& b) { return F::mul(a, b); }
    static HD T cmul(const T& a, const T& c) { return F::mul(a, c); }
    static HD T konst(const T& a) { return F::load(a); }
    static HD T kone() { return F::one(); }
    static HD T kmul(const T& a, const T& b) { return F::mul(a, b); }
    static HD T inv(const T& a) { return F::inv(a); }
};
// Goldilocks: data are plain canonical words, constants are kept times 2^64 (see ff/gl64.cuh) so
// that data * constant is a single multiplication-free-reduction product
template<> struct arith<gl64> {
    typedef uint64_t T;
    static HD T zero() { return 0; }
    static HD T one() { return 1; }
    static HD T load(T a) { return gl64::canon(a); }
    static HD T add(T a, T b) { return gl64::canon(gl64::add(a, b)); }
    static HD T dmul(T a, T b) { return gl64::mul_plain(a, b); }
    static HD T cmul(T a, T c) { return gl64::mul(a, c); }
    static HD T konst(T a) { return gl64::to_mont(a); }
    static HD T kone() { return gl64::one(); }
    static HD T kmul(T a, T b) { return gl64::mul(a, b); }
    static HD T inv(T a) { return gl64::mul(gl64::pow(gl64::to_mont(a), gl64::P - 2), 1); }
};

HD bool is_zero(uint32_t a) { return a == 0; }
HD bool is_zero(uint64_t a) { return a == 0; }
template<class T> HD bool is_zero(const T& a)
{
    uint32_t acc = 0;
#pragma unroll
    for (size_t i = 0; i < sizeof(a.l) / sizeof(a.l[0]); i++) acc |= a.l[i];
    return acc == 0;
}

template<class F> HD typename F::T kpow(typename F::T c, uint64_t e)
{
    typedef arith<F> A;
    typename F::T r = A::kone();
    for (; e; e >>= 1, c = A::kmul(c, c))
        if (e & 1) r = A::kmul(r, c);
    return r;
}

// The powers of z a division needs, computed ONCE on the host (about 130 field multiplications)
// and handed to the kernels by value: a carry that crosses k elements is weighted by z^k, and every
// level of the scan hierarchy spans a fixed number of elements.  Unused by Add / Multiply.
template<class T, int E, int BS> struct scan_tab {
    static constexpr int NW = BS / 32;
    T wl[33];          // z^(E k): crossing k threads
    T ww[NW + 1];      // z^(32 E k): crossing k warps
    T zp[E + 1];       // z^k
    T zt;              // z^TILE, TILE = BS E
    T zw[10];          // z^(2^k): weights of the reduce pass's tree
    T y;               // z^BS
    T tw[10];          // zt^(2^k), and
    T yt;              // zt^BS: folding tile aggregates (MODE_COOP)
};
template<class F, int E, int BS>
inline void scan_tab_fill(scan_tab<typename F::T, E, BS>& t, const typename F::T& z)
{
    typedef arith<F> A;
    constexpr int NW = BS / 32;
    t.zp[0] = A::kone();
    for (int k = 1; k <= E; k++) t.zp[k] = A::kmul(t.zp[k - 1], z);
    t.wl[0] = A::kone();
    for (int k = 1; k <= 32; k++) t.wl[k] = A::kmul(t.wl[k - 1], t.zp[E]);
    t.ww[0] = A::kone();
    for (int k = 1; k <= NW; k++) t.ww[k] = A::kmul(t.ww[k - 1], t.wl[32]);
    t.zt = t.ww[NW];
    t.zw[0] = z;
    for (int k = 1; k < 10; k++) t.zw[k] = A::kmul(t.zw[k - 1], t.zw[k - 1]);
    t.y = kpow<F>(z, BS);
    t.tw[0] = t.zt;
    for (int k = 1; k < 10; k++) t.tw[k] = A::kmul(t.tw[k - 1], t.tw[k - 1]);
    t.yt = kpow<F>(t.zt, BS);
}

#if defined(__CUDACC__)
// ---- whole-element warp shuffles and L2 loads (role of the reference's ff/shfl.cuh) --------------
DEV uint32_t shfl_up(uint32_t v, uint32_t d) { return __shfl_up_sync(0xffffffffu, v, d); }
DEV uint64_t shfl_up(uint64_t v, uint32_t d) { return __shfl_up_sync(0xffffffffu, v, d); }
DEV uint32_t shfl_down(uint32_t v, uint32_t d) { return __shfl_down_sync(0xffffffffu, v, d); }
DEV uint64_t shfl_down(uint64_t v, uint32_t d) { return __shfl_down_sync(0xffffffffu, v, d); }
DEV uint32_t shfl_idx(uint32_t v, uint32_t l) { return __shfl_sync(0xffffffffu, v, l); }
DEV uint64_t shfl_idx(uint64_t v, uint32_t l) { return __shfl_sync(0xffffffffu, v, l); }
template<class T> DEV T shfl_up(const T& v, uint32_t d)
{
    T r;
#pragma unroll
    for (size_t i = 0; i < sizeof(v.l) / 4; i++) r.l[i] = __shfl_up_sync(0xffffffffu, v.l[i], d);
    return r;
}
template<class T> DEV T shfl_down(const T& v, uint32_t d)
{
    T r;
#pragma unroll
    for (size_t i = 0; i < sizeof(v.l) / 4; i++) r.l[i] = __shfl_down_sync(0xffffffffu, v.l[i], d);
    return r;
}
template<class T> DEV T shfl_idx(const T& v, uint32_t l)
{
    T r;
#pragma unroll
    for (size_t i = 0; i < sizeof(v.l) / 4; i++) r.l[i] = __shfl_sync(0xffffffffu, v.l[i], l);
    return r;
}
DEV uint32_t ld_cg(const uint32_t* p) { return __ldcg(p); }
DEV uint64_t ld_cg(const uint64_t* p) { return __ldcg((const unsigned long long*)p); }
template<class T> DEV T ld_cg(const T* p)
{
    static_assert(sizeof(T) % 16 == 0, "wide elements are 16-byte multiples");
    T r;
    const uint4* q = (const uint4*)p;
#pragma unroll
    for (size_t i = 0; i < sizeof(T) / 16; i++) ((uint4*)&r)[i] = __ldcg(q + i);
    return r;
}

enum { OP_ADD = 0, OP_MUL = 1, OP_DIV = 2 };

// carry (what precedes, in scan order) joined with x; w = z^(number of elements x spans), OP_DIV only
template<class F, int OP> DEV typename F::T join(const typename F::T& carry, const typename F::T& x,
                                                 const typename F::T& w)
{
    typedef arith<F> A;
    if (OP == OP_ADD) return A::add(carry, x);
    if (OP == OP_MUL) return A::dmul(carry, x);
    return A::add(x, A::cmul(carry, w));
}

// ---- sum_t val_t * base^t over the CTA (thread 0 holds the result) ---------------------------------
// weights base^(2^k), k < 10, once per base ...
template<class F>
DEV void wreduce_setup(const typename F::T& base, typename F::T* s_w /*[10]*/)
{
    typedef arith<F> A;
    __syncthreads();                                            // s_w free again
    if (threadIdx.x < 10) {
        typename F::T b = base;
        for (uint32_t i = 0; i < threadIdx.x; i++) b = A::kmul(b, b);
        s_w[threadIdx.x] = b;
    }
    __syncthreads();
}
// ... then any number of reductions with them
template<class F, int BS>
DEV typename F::T wreduce(typename F::T val, const typename F::T* s_w, typename F::T* s_x /*[BS/32]*/)
{
    typedef arith<F> A;
    typedef typename F::T T;
    constexpr int NW = BS / 32;
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
#pragma unroll
    for (uint32_t k = 0, off = 1; off < 32; k++, off <<= 1) {
        T t = shfl_down(val, off);
        val = A::add(val, A::cmul(t, s_w[k]));
    }
    __syncthreads();                                            // s_x free again
    if (lane == 0) s_x[warp] = val;
    __syncthreads();
    if (warp == 0) {
        val = lane < NW ? s_x[lane] : A::zero();
#pragma unroll
        for (uint32_t k = 5, off = 1; off < NW; k++, off <<= 1) {
            T t = shfl_down(val, off);
            val = A::add(val, A::cmul(t, s_w[k]));
        }
    }
    return val;
}
template<class F, int BS>
DEV typename F::T block_wreduce(typename F::T val, const typename F::T& base, typename F::T* s_w, typename F::T* s_x)
{
    wreduce_setup<F>(base, s_w);
    return wreduce<F, BS>(val, s_w, s_x);
}

// ---- scan -------------------------------------------------------------------------------------------
// Scan order t = 0, 1, ...: memory index t, or len-1-t when `rev` (division walks down from the top
// coefficient).  Thread = E consecutive scan positions, warp = 32 E, tile = BS E; a warp moves its
// 32 E elements between memory and registers through a padded shared-memory transpose, so global
// accesses are contiguous per warp in either direction.  The last tile may be ragged (its tail is
// the identity and is not stored).
//
// Three launches make a scan of any length, with no ordering between CTAs:
//   tile_reduce_kernel        every tile's aggregate -> aggs[tile]                      (reads the data once)
//   scan_kernel MODE_SERIAL   ONE CTA scans aggs[] in place, tile after tile            (ntiles elements)
//   scan_kernel MODE_SCAN     every tile rescanned with carry aggs[tile-1] and stored   (reads + writes the data)
// A decoupled look-back single pass was tried first and rejected: its carry chain advances at most
// one 32-tile window per L2 round trip, where these three launches are bandwidth bound.  Short
// inputs take MODE_SERIAL
// directly on the data (one launch).  Inputs whose tiles are all resident at once take MODE_COOP:
// one cooperative launch, one tile per CTA kept in registers across a single grid barrier, after
// which every CTA folds the aggregates of the tiles before it by itself (a few KB from L2) -- one
// read and one write of the data and a third of the launch latency, which is what mid sizes cost.
enum { MODE_SERIAL = 1, MODE_SCAN = 2, MODE_COOP = 3 };

// MODE_COOP: what precedes tile `tile`, from the aggregates of tiles 0 .. tile-1 (thread 0 holds it).
// Division: sum_j aggs[tile-1-j] * zt^j, thread t taking j = t, t+BS, ... by Horner in zt^BS.
template<class F, int OP, int BS>
DEV typename F::T carry_from_aggs(const typename F::T* aggs, uint32_t tile, const typename F::T& yt,
                                  const typename F::T* s_w, typename F::T* s_x)
{
    typedef arith<F> A;
    typedef typename F::T T;
    constexpr int NW = BS / 32;
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const T ident = OP == OP_MUL ? A::one() : A::zero();
    T acc = ident;
    if (OP == OP_DIV) {
        if (tid < tile) {
            for (uint32_t j = tid + (tile - 1 - tid) / BS * BS;; j -= BS) {      // largest j = tid (mod BS) below tile
                acc = A::add(A::cmul(acc, yt), ld_cg(aggs + (tile - 1 - j)));
                if (j < BS) break;
            }
        }
        return wreduce<F, BS>(acc, s_w, s_x);
    }
    for (uint32_t i = tid; i < tile; i += BS) acc = join<F, OP>(acc, ld_cg(aggs + i), yt);
#pragma unroll
    for (uint32_t off = 16; off; off >>= 1) acc = join<F, OP>(acc, shfl_down(acc, off), yt);
    __syncthreads();
    if (lane == 0) s_x[warp] = acc;
    __syncthreads();
    if (warp == 0) {
        acc = lane < NW ? s_x[lane] : ident;
#pragma unroll
        for (uint32_t off = NW / 2; off; off >>= 1) acc = join<F, OP>(acc, shfl_down(acc, off), yt);
    }
    return acc;
}

template<class F, int OP, int E, int BS, int MODE, bool REV>
__global__ __launch_bounds__(BS) void scan_kernel(typename F::T* out, const typename F::T* in, size_t len,
                                                  const __grid_constant__ scan_tab<typename F::T, E, BS> tab,
                                                  int rotate, uint32_t ntiles,
                                                  typename F::T* aggs, typename F::T* edge)
{
    typedef arith<F> A;
    typedef typename F::T T;
    constexpr int NW = BS / 32;
    constexpr uint32_t TILE = BS * E;
    constexpr int ROW = E + 1;       // padded row of the transpose
    static_assert(NW <= 32 && (E & (E - 1)) == 0, "one warp scans the warp aggregates; E is a power of two");
    __shared__ scan_tab<T, E, BS> s_tab;
    __shared__ T s_agg[NW];
    __shared__ T s_carry;
    __shared__ T s_stage[NW][32 * ROW];
    __shared__ T s_x2[NW];
    const T* const s_wl = s_tab.wl;
    const T* const s_ww = s_tab.ww;
    const T* const s_zp = s_tab.zp;

    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const T ident = OP == OP_MUL ? A::one() : A::zero();

    if (OP == OP_DIV)
        for (uint32_t i = tid; i < sizeof(tab) / sizeof(T); i += BS) ((T*)&s_tab)[i] = ((const T*)&tab)[i];
    if (tid == 0) s_carry = ident;
    const T z = OP == OP_DIV ? tab.zp[1] : ident;

    // element e = j*32 + lane of the warp's 32 E sits at stage[sidx + j * SJ] (row e / E, column e % E)
    const uint32_t sidx = (lane / E) * ROW + lane % E;
    constexpr uint32_t SJ = (32 / E) * ROW;
    static_assert(E <= 32, "a warp's stripe of 32 elements covers whole rows");

    for (uint32_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        __syncthreads();            // constants ready; previous tile's s_agg / s_stage consumed
        const size_t tbase = (size_t)tile * TILE;
        const uint32_t wofs = warp * 32 * E;
        const bool full = tbase + TILE <= len;
        T cprev = ident;
        if (MODE == MODE_SCAN && tid == 0 && tile) cprev = ld_cg(aggs + tile - 1);
        T* stage = s_stage[warp];
        if (full) {                 // scan position tbase + wofs + e  <->  memory index, no bounds to check
            const T* src = REV ? in + (len - 1 - tbase - wofs - lane) : in + (tbase + wofs + lane);
#pragma unroll
            for (int j = 0; j < E; j++) stage[sidx + j * SJ] = A::load(REV ? *(src - j * 32) : src[j * 32]);
        } else {
#pragma unroll
            for (int j = 0; j < E; j++) {
                const size_t pos = tbase + wofs + j * 32 + lane;
                T c = ident;
                if (pos < len) c = A::load(in[REV ? len - 1 - pos : pos]);
                stage[sidx + j * SJ] = c;
            }
        }
        __syncwarp();
        T v[E];
#pragma unroll
        for (int j = 0; j < E; j++) v[j] = stage[lane * ROW + j];
#pragma unroll
        for (int j = 1; j < E; j++) v[j] = join<F, OP>(v[j - 1], v[j], z);

        T inc = v[E - 1];
#pragma unroll
        for (uint32_t off = 1; off < 32; off <<= 1) {
            T t = shfl_up(inc, off);
            if (lane >= off) inc = join<F, OP>(t, inc, s_wl[off]);
        }
        T lane_excl = shfl_up(inc, 1);
        if (lane == 0) lane_excl = ident;
        if (lane == 31) s_agg[warp] = inc;
        __syncthreads();

        if (warp == 0) {
            T w = lane < NW ? s_agg[lane] : ident;
#pragma unroll
            for (uint32_t off = 1; off < NW; off <<= 1) {
                T t = shfl_up(w, off);
                if (lane >= off) w = join<F, OP>(t, w, s_ww[off]);
            }
            if (lane < NW) s_agg[lane] = w;
            if (MODE == MODE_SCAN && lane == 0) s_carry = cprev;
            if (MODE == MODE_COOP && lane == NW - 1) aggs[tile] = w;
        }
        if (MODE == MODE_COOP) {    // every tile is in registers somewhere: one barrier, then each CTA for itself
            __threadfence();
            cooperative_groups::this_grid().sync();
            const T c = carry_from_aggs<F, OP, BS>(aggs, tile, s_tab.yt, s_tab.tw, s_x2);
            if (tid == 0) s_carry = c;
        }
        __syncthreads();

        const T carry = s_carry;
        const T wexcl = warp ? s_agg[warp - 1] : ident;
        const T wc = join<F, OP>(carry, wexcl, s_ww[warp]);            // value entering this warp
        const T cin = join<F, OP>(wc, lane_excl, s_wl[lane]);          // value entering this thread
#pragma unroll
        for (int j = 0; j < E; j++) stage[lane * ROW + j] = join<F, OP>(cin, v[j], s_zp[j + 1]);
        if (MODE == MODE_SERIAL) {
            __syncthreads();                                           // every thread has read s_carry
            if (tid == BS - 1) s_carry = stage[lane * ROW + E - 1];    // inclusive value at the tile's end
        }
        __syncwarp();
        if (full && !(REV && rotate)) {
            T* dst = REV ? out + (len - 1 - tbase - wofs - lane) : out + (tbase + wofs + lane);
#pragma unroll
            for (int j = 0; j < E; j++) {
                if (REV) *(dst - j * 32) = stage[sidx + j * SJ];
                else dst[j * 32] = stage[sidx + j * SJ];
            }
        } else if (full && tile + 1 < ntiles) {
            // rotate, interior tile: every quotient coefficient moves one slot down; the last one
            // would land in the next tile's still unread first slot and is parked instead
            T* dst = out + (len - 2 - tbase - wofs - lane);
#pragma unroll
            for (int j = 0; j < E; j++) {
                const T r = stage[sidx + j * SJ];
                if (MODE != MODE_COOP && j == E - 1 && tid == BS - 1) edge[tile] = r;   // (COOP: all tiles were read)
                else *(dst - j * 32) = r;
            }
        } else {
#pragma unroll
            for (int j = 0; j < E; j++) {
                const uint32_t e = j * 32 + lane;
                const size_t pos = tbase + wofs + e;
                if (pos >= len) continue;
                const T r = stage[sidx + j * SJ];
                if (!REV) out[pos] = r;
                else if (!rotate) out[len - 1 - pos] = r;
                else if (pos == len - 1) out[len - 1] = r;             // the remainder goes last
                else if (MODE != MODE_COOP && e == 32 * E - 1 && warp == NW - 1) edge[tile] = r;
                else out[len - 2 - pos] = r;
            }
        }
    }
}

// The first of the three launches: a tile's aggregate needs no per-element prefix, so thread t takes
// the tile's positions t, t+BS, ... (contiguous per warp, no transpose).  Add / Multiply fold them
// in any order; division runs Horner in z^BS over its positions (mirrored, so that thread t ends up
// weighted by z^t) and finishes with the weighted tree above: one multiplication per element.
template<class F, int OP, int E, int BS>
__global__ __launch_bounds__(BS) void tile_reduce_kernel(typename F::T* aggs, const typename F::T* in, size_t len,
                                                         const __grid_constant__ scan_tab<typename F::T, E, BS> tab,
                                                         int rev, uint32_t ntiles)
{
    typedef arith<F> A;
    typedef typename F::T T;
    constexpr int NW = BS / 32;
    constexpr uint32_t TILE = BS * E;
    __shared__ T s_w[10];
    __shared__ T s_x[NW];
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const T ident = OP == OP_MUL ? A::one() : A::zero();
    if (OP == OP_DIV) {
        if (tid < 10) s_w[tid] = tab.zw[tid];
        __syncthreads();
    }
    const T y = OP == OP_DIV ? tab.y : ident;
    for (uint32_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const size_t base = (size_t)tile * TILE + (OP == OP_DIV ? BS - 1 - tid : tid);
        T acc = ident;
        if ((size_t)(tile + 1) * TILE <= len) {
            const T* src = rev ? in + (len - 1 - base) : in + base;
            const ptrdiff_t step = rev ? -(ptrdiff_t)BS : (ptrdiff_t)BS;
#pragma unroll
            for (int k = 0; k < E; k++) acc = join<F, OP>(acc, A::load(src[k * step]), y);
        } else {
#pragma unroll
            for (int k = 0; k < E; k++) {
                const size_t pos = base + (size_t)k * BS;
                T c = ident;
                if (pos < len) c = A::load(in[rev ? len - 1 - pos : pos]);
                acc = join<F, OP>(acc, c, y);
            }
        }
        if (OP == OP_DIV) {
            acc = wreduce<F, BS>(acc, s_w, s_x);
        } else {
#pragma unroll
            for (uint32_t off = 16; off; off >>= 1) acc = join<F, OP>(acc, shfl_down(acc, off), y);
            __syncthreads();
            if (lane == 0) s_x[warp] = acc;
            __syncthreads();
            if (warp == 0) {
                acc = lane < NW ? s_x[lane] : ident;
#pragma unroll
                for (uint32_t off = NW / 2; off; off >>= 1) acc = join<F, OP>(acc, shfl_down(acc, off), y);
            }
        }
        if (tid == 0) aggs[tile] = acc;
    }
}

// rotate=true: the quotient coefficient at a tile's last scan position lands in the first input
// slot of the NEXT tile, which that tile may not have read yet; it is parked and stored here
template<class T>
__global__ void scan_edge_kernel(T* out, const T* edge, size_t len, uint32_t ntiles, uint32_t tile_elems)
{
    uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k + 1 >= ntiles) return;
    size_t pos = (size_t)(k + 1) * tile_elems - 1;
    out[len - 2 - pos] = edge[k];
}

// one partial per (point, CTA).  Thread g of the G = gridDim.x*BS threads owns the coefficients
// g, g+G, g+2G, ... (a warp reads consecutive elements) and runs Horner over them in y = x^G:
// one multiplication per coefficient and point; then  sum_t s_t x^t  over the CTA.  PTS points share
// one pass over the coefficients.
template<class F, int BS, int PTS>
__global__ __launch_bounds__(BS) void evaluate_partial_kernel(typename F::T* partial, const typename F::T* x,
                                                              uint32_t npoints, const typename F::T* coeffs,
                                                              size_t len)
{
    typedef arith<F> A;
    typedef typename F::T T;
    __shared__ T s_w[10];
    __shared__ T s_x[BS / 32];
    __shared__ T s_y[PTS], s_xk[PTS];
    const size_t G = (size_t)gridDim.x * BS, g = (size_t)blockIdx.x * BS + threadIdx.x;
    const size_t rows = (len + G - 1) / G;
    for (uint32_t p0 = 0; p0 < npoints; p0 += PTS) {
        __syncthreads();
        if (threadIdx.x < PTS && p0 + threadIdx.x < npoints) {
            s_xk[threadIdx.x] = A::konst(x[p0 + threadIdx.x]);
            s_y[threadIdx.x] = kpow<F>(s_xk[threadIdx.x], G);
        }
        __syncthreads();
        T y[PTS], s[PTS];
#pragma unroll
        for (int q = 0; q < PTS; q++) {
            y[q] = s_y[p0 + q < npoints ? q : 0];
            s[q] = A::zero();
        }
#pragma unroll 4
        for (size_t k = rows; k-- > 0;) {
            const size_t idx = k * G + g;
            T c = A::zero();
            if (idx < len) c = A::load(coeffs[idx]);
#pragma unroll
            for (int q = 0; q < PTS; q++) s[q] = A::add(A::cmul(s[q], y[q]), c);
        }
        for (int q = 0; q < PTS && p0 + q < npoints; q++) {
            T r = block_wreduce<F, BS>(s[q], s_xk[q], s_w, s_x);
            if (threadIdx.x == 0) partial[(size_t)(p0 + q) * gridDim.x + blockIdx.x] = r;
        }
    }
}

// ret[p] = sum_k partial[p][k] * (x^tile_elems)^k, one CTA per point
template<class F, int BS>
__global__ __launch_bounds__(BS) void evaluate_finish_kernel(typename F::T* ret, const typename F::T* partial,
                                                             const typename F::T* x, uint32_t nparts,
                                                             uint32_t tile_elems)
{
    typedef arith<F> A;
    typedef typename F::T T;
    __shared__ T s_w[10];
    __shared__ T s_x[BS / 32];
    const uint32_t p = blockIdx.x, per = (nparts + BS - 1) / BS;
    const T xt = kpow<F>(A::konst(x[p]), tile_elems);
    const T* mine = partial + (size_t)p * nparts;
    T s = A::zero();
    for (uint32_t j = per; j-- > 0;) {
        uint32_t k = threadIdx.x * per + j;
        s = A::cmul(s, xt);
        if (k < nparts) s = A::add(s, mine[k]);
    }
    T r = block_wreduce<F, BS>(s, kpow<F>(xt, per), s_w, s_x);
    if (threadIdx.x == 0) ret[p] = r;
}

// ---- batch inversion -------------------------------------------------------------------------------
// ff/batch_inversion.hpp:14-51 for a caller's own kernel: out[i] = 1/inp[i], zero where inp[i] is
// zero, one field inversion for the N elements (Montgomery's trick; zeros are stepped over by
// multiplying with one instead, the reference's csel/czero)
template<class F, int N>
DEV void batch_inversion(typename F::T out[N], const typename F::T inp[N])
{
    typedef arith<F> A;
    typedef typename F::T T;
    T acc = A::one();
#pragma unroll
    for (int i = 0; i < N; i++) {
        out[i] = acc;                                          // product of what precedes
        acc = A::dmul(acc, is_zero(inp[i]) ? A::one() : inp[i]);
    }
    T inv = A::inv(acc);
#pragma unroll
    for (int i = N - 1; i >= 0; i--) {
        const bool zero = is_zero(inp[i]);
        T next = A::dmul(inv, zero ? A::one() : inp[i]);
        out[i] = zero ? A::zero() : A::dmul(inv, out[i]);
        inv = next;
    }
}

// the array form: every CTA shares one inversion among its BS*N elements (INV_SELF).  The inversion
// is a serial chain of a few hundred multiplications run by ONE warp, so for long arrays of wide
// elements it is hoisted out: INV_PRODUCT writes each chunk's product to tots[], the host inverts
// tots[] with this same routine (recursively, a 2048-fold smaller array), and INV_GIVEN finishes
// with the chunk inverses read back -- four multiplications per element and nothing serial.
enum { INV_SELF = 0, INV_PRODUCT = 1, INV_GIVEN = 2 };
template<class F, int N, int BS, int MODE>
__global__ __launch_bounds__(BS) void batch_inverse_kernel(typename F::T* out, const typename F::T* in, size_t len,
                                                           typename F::T* tots)
{
    typedef arith<F> A;
    typedef typename F::T T;
    constexpr int NW = BS / 32;
    __shared__ T s_agg[NW], s_pre[NW], s_suf[NW];
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const size_t nchunks = (len + (size_t)BS * N - 1) / ((size_t)BS * N);

    for (size_t chunk = blockIdx.x; chunk < nchunks; chunk += gridDim.x) {
        const size_t base = (chunk * BS + tid) * N;
        T x[N], pre[N];
        T a = A::one();
#pragma unroll
        for (int i = 0; i < N; i++) {
            x[i] = A::one();
            if (base + i < len) x[i] = A::load(in[base + i]);
            pre[i] = a;
            a = A::dmul(a, is_zero(x[i]) ? A::one() : x[i]);
        }
        // product of every OTHER thread's chunk = (lanes before) (lanes after) (warps before) (warps after)
        T pi = a, si = a;
#pragma unroll
        for (uint32_t off = 1; off < 32; off <<= 1) {
            T t = shfl_up(pi, off);
            if (lane >= off) pi = A::dmul(t, pi);
            T u = shfl_down(si, off);
            if (lane + off < 32) si = A::dmul(u, si);
        }
        T before = shfl_up(pi, 1), after = shfl_down(si, 1);
        if (lane == 0) before = A::one();
        if (lane == 31) after = A::one();
        __syncthreads();                                        // previous chunk's s_* consumed
        if (lane == 31) s_agg[warp] = pi;
        __syncthreads();
        if (warp == 0) {
            T wa = lane < NW ? s_agg[lane] : A::one();
            T wp = wa, ws = wa;
#pragma unroll
            for (uint32_t off = 1; off < 32; off <<= 1) {
                T t = shfl_up(wp, off);
                if (lane >= off) wp = A::dmul(t, wp);
                T u = shfl_down(ws, off);
                if (lane + off < 32) ws = A::dmul(u, ws);
            }
            if (MODE == INV_PRODUCT) {
                if (lane == 31) tots[chunk] = wp;
                continue;
            }
            const T total_inv = MODE == INV_GIVEN ? ld_cg(tots + chunk) : A::inv(shfl_idx(wp, 31));   // the one inversion
            T wb = shfl_up(wp, 1), wf = shfl_down(ws, 1);
            if (lane == 0) wb = A::one();
            if (lane == 31) wf = A::one();
            if (lane < NW) {
                s_pre[lane] = wb;
                s_suf[lane] = A::dmul(wf, total_inv);
            }
        }
        if (MODE == INV_PRODUCT) continue;
        __syncthreads();
        T inv = A::dmul(A::dmul(before, after), A::dmul(s_pre[warp], s_suf[warp]));   // 1 / a
#pragma unroll
        for (int i = N - 1; i >= 0; i--) {
            const bool zero = is_zero(x[i]);
            T r = zero ? A::zero() : A::dmul(inv, pre[i]);
            inv = A::dmul(inv, zero ? A::one() : x[i]);
            if (base + i < len) out[base + i] = r;
        }
    }
}
#endif  // __CUDACC__

}  // namespace poly
