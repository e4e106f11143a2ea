// NTT pass machinery for single-word fields (gl64, bb31).
//
// An N = 2^n point NTT is executed as P <= 3 "passes".  A pass is one kernel launch in
// which every CTA owns a tile of W independent columns x 2^R rows, pulls it from HBM into
// shared memory, runs a complete 2^R-point sub-NTT on each column there (radix-2 DIT
// butterflies, 16 elements per thread in registers between shared-memory exchanges, XOR-swizzled rows),
// applies the inter-pass twiddle w_N^(row*col) and writes the tile back.  Every element
// is therefore read and written exactly once per pass: algorithmic traffic per pass is
// 2*N*sizeof(T) and a 2^24 transform needs two passes (the reference needs three
// <=10-stage steps plus a bit-reversal pass for the same NN transform,
// ntt/ntt.cuh:100-127,174-178).
//
// The four orders of the reference API (ntt/ntt.cuh:33,174-194) are four ways of
// assigning index digits to passes; they share this kernel and differ only in the
// host-built descriptor (ntt_plan.hpp):
//   NR  in place, top digit first,    digit left bit-reversed,  twiddle at store
//   RN  in place, bottom digit first, digit arrives bit-reversed, twiddle at load
//   NN  ping-pong through a scratch buffer, strided gather -> transposed scatter
//   RR  mirror image of NN
//
// Everything here is HD (host+device) so tests/emu/ntt_emu.cpp can run the same code
// phase by phase on the CPU; the shipped path is ntt.cu (CUDA only).
#pragma once
#include "../util/hd.cuh"

namespace ntt {

constexpr uint32_t LG_DENSE = 12;        // largest sub-NTT: 2^12 rows
// elements per thread per register step = 2^F::LG_EPT: 16 for the one-word fields (32 live
// registers of data), 4 for the 256-bit Montgomery fields (8 words each)
constexpr uint32_t LG_TLO = 12;          // low half of the two-level w_N^e table

enum TwMode : uint32_t { TW_NONE = 0, TW_LOAD = 1, TW_STORE = 2 };

struct Pass {
    uint32_t lg_r;                       // rows   = 2^lg_r  (sub-NTT length)
    uint32_t lg_w;                       // columns = 2^lg_w (independent sub-NTTs per tile)
    // element address = th*(t >> lg_tlo) + tl*(t & mask) + (row << lg_sa) + (col << lg_sc)
    uint32_t in_lg_tlo, in_lg_sa, in_lg_sc;
    uint64_t in_tl, in_th;
    uint32_t out_lg_tlo, out_lg_sa, out_lg_sc;
    uint64_t out_tl, out_th;
    uint32_t in_rev;                     // rows arrive in bit-reversed order
    uint32_t out_rev;                    // rows leave in bit-reversed order
    uint32_t tw_mode, tw_rsh, tw_bits, tw_brev, tw_lsh;
    uint32_t scale;                      // multiply by n^-1 at store (last pass of an inverse)
    uint32_t src, dst;                   // 0 = caller's buffer, 1 = scratch
    // slab-sharded transforms only (zero otherwise): the output row index is split, its top
    // bits select the destination rank's block of the all-to-all staging buffer; and the
    // twiddle column is offset by the first column this rank owns
    uint32_t out_split_bits, out_split_shift;
    uint32_t tw_col_offset;
    // fused exchange (peer_on != 0): the store goes straight into the RECEIVING rank's buffer over
    // NVLink instead of a local staging block: destination q = row >> peer_shift, address =
    // peer[q] + peer_block (this sender's block in every receiver) + tile/row/column offsets
    uint32_t peer_on, peer_shift;
    uint64_t peer_block;
    uint64_t peer[8];
};

// coset factor of element i of a batch of 2^lg_n-point transforms: g^e, e = the element's
// position within its transform, bit-reversed if `bitrev`; g0/g1/g2 hold g^i, g^(i << 12),
// g^(i << 24)
template<class F>
HD typename F::T coset_mul(typename F::T x, uint64_t i, uint32_t lg_n, bool bitrev,
                           const typename F::T* g0, const typename F::T* g1, const typename F::T* g2)
{
    const uint32_t j = (uint32_t)i & ((1u << lg_n) - 1), e = bitrev ? brev32(j, lg_n) : j;
    x = F::mul(x, g0[e & 4095]);
    if (e >> 12) x = F::mul(x, g1[(e >> 12) & 4095]);
    if (e >> 24) x = F::mul(x, g2[e >> 24]);
    return x;
}

template<class F> struct Tables {
    const typename F::T* dense;          // dense[h + i] = w_(2h)^i, h = 1,2,4..2^(LG_DENSE-1)
    const typename F::T* tlo;            // tlo[i] = w_N^i,            i < 2^LG_TLO
    const typename F::T* thi;            // thi[i] = w_N^(i << LG_TLO)
    typename F::T ninv;                  // 2^-n
    // warp-autonomous passes (ntt_warp.cuh): twist tables of the 2^5..2^8-point sub-NTTs,
    // mid[mid_offset(R) + k0 * 2^(R-4) + b] = w_(2^R)^(b * k0), and the powers of w_16
    const typename F::T* mid;
    typename F::T w16[8];
};

// ---- compile-time / run-time views of the shape of a pass ------------------------------
// The phase functions read the tile shape through a "knobs" object.  KDyn forwards to the
// descriptor (any shape, slower index arithmetic); KStat<...> fixes the shape at compile time
// so that every shift, mask, bit-reversal width and loop bound folds into an immediate.  The
// hot shapes produced by the planner are instantiated statically in ntt.cu.
struct KDyn {
    const Pass& d;
    HD uint32_t lg_r() const { return d.lg_r; }
    HD uint32_t lg_w() const { return d.lg_w; }
    HD bool in_row_fast() const { return d.in_lg_sa == 0; }
    HD bool out_row_fast() const { return d.out_lg_sa == 0; }
    HD bool in_rev() const { return d.in_rev != 0; }
    HD bool out_rev() const { return d.out_rev != 0; }
    HD uint32_t tw_mode() const { return d.tw_mode; }
};
template<uint32_t R, uint32_t W, bool IRF, bool ORF, bool IREV, bool OREV, uint32_t TW>
struct KStat {
    HD explicit KStat(const Pass&) {}
    static HD constexpr uint32_t lg_r() { return R; }
    static HD constexpr uint32_t lg_w() { return W; }
    static HD constexpr bool in_row_fast() { return IRF; }
    static HD constexpr bool out_row_fast() { return ORF; }
    static HD constexpr bool in_rev() { return IREV; }
    static HD constexpr bool out_rev() { return OREV; }
    static HD constexpr uint32_t tw_mode() { return TW; }
};
// tile shape fixed at compile time, order and twiddle flags read from the descriptor (the matrix
// passes: one instantiation per shape serves every order)
template<uint32_t R, uint32_t W>
struct KShape {
    const Pass& d;
    HD explicit KShape(const Pass& d_) : d(d_) {}
    static HD constexpr uint32_t lg_r() { return R; }
    static HD constexpr uint32_t lg_w() { return W; }
    HD bool in_rev() const { return d.in_rev != 0; }
    HD bool out_rev() const { return d.out_rev != 0; }
    HD uint32_t tw_mode() const { return d.tw_mode; }
};

// Shared-memory placement of row `i` of column `c`: an XOR swizzle of the low four index bits
// with bits 4-7, bits 8-11 and the column, so that a half-warp (sixteen 8-byte words = all 32
// banks) is conflict-free for every access pattern of a pass: sixteen consecutive rows
// (register steps with stride >= 16, natural-order tile I/O), sixteen rows 16 apart (the
// stride-1 register step), sixteen rows 2^(R-4) apart (bit-reversed tile I/O), and rows x
// columns mixes (strided tile I/O).  No padding: a column is exactly 2^R words.
HD uint32_t swz(uint32_t i, uint32_t c, uint32_t lg_r)
{
    return i ^ (((i >> 4) ^ (i >> 8) ^ c) & (lg_r >= 4 ? 15u : (1u << lg_r) - 1));
}
HD uint32_t col_stride(uint32_t lg_r) { return 1u << lg_r; }
template<class F> HD uint32_t tile_threads(const Pass& d)
{
    return (d.lg_r >= F::LG_EPT ? (1u << (d.lg_r - F::LG_EPT)) : 1u) << d.lg_w;
}
HD uint32_t smem_elems(const Pass& d) { return (col_stride(d.lg_r) << d.lg_w) + (1u << d.lg_r); }

HD uint64_t tile_base(uint32_t t, uint32_t lg_tlo, uint64_t tl, uint64_t th)
{
    uint32_t lo = lg_tlo >= 32 ? t : (t & ((1u << lg_tlo) - 1));
    uint32_t hi = lg_tlo >= 32 ? 0 : (t >> lg_tlo);
    return tl * lo + th * hi;
}

template<class F> HD typename F::T twiddle(const Tables<F>& tb, uint32_t e)
{
    typename F::T lo = tb.tlo[e & ((1u << LG_TLO) - 1)];
    uint32_t h = e >> LG_TLO;
    return h ? F::mul(lo, tb.thi[h]) : lo;
}

HD uint32_t tw_column_value(const Pass& d, uint64_t pos0)
{
    uint32_t v = (uint32_t)(pos0 >> d.tw_rsh) & (d.tw_bits >= 32 ? ~0u : ((1u << d.tw_bits) - 1));
    return (d.tw_brev ? brev32(v, d.tw_bits) : v) + d.tw_col_offset;
}

#if defined(__CUDACC__)
// ---- TMA (bulk asynchronous copy) of a twiddle table into shared memory -------------------------
// One thread arms an mbarrier with the byte count and issues ONE cp.async.bulk (SASS: UBLKCP): the
// copy engine of the SM moves the table while all threads go on (here: into the first tile load);
// consumers wait on the barrier's phase before their first table read.
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t arrivals)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_u32(bar)), "r"(arrivals) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void tma_load_1d(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_u32(bar)), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 :: "r"(smem_u32(smem_dst)), "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity)
{
    asm volatile("{\n\t.reg .pred p;\n\t"
                 "MBAR_WAIT:\n\t"
                 "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
                 "@p bra MBAR_DONE;\n\t"
                 "bra MBAR_WAIT;\n\t"
                 "MBAR_DONE:\n\t}" :: "r"(smem_u32(bar)), "r"(parity) : "memory");
}
#endif

// ---- phase 0: per-CTA copy of the sub-NTT twiddles into shared memory -------------
template<class F, class K>
HD void phase_twiddles(const K k, const Tables<F>& tb, typename F::T* smem,
                       uint32_t tid, uint32_t nthreads)
{
    typename F::T* tw = smem + (col_stride(k.lg_r()) << k.lg_w());
    for (uint32_t i = tid; i < (1u << k.lg_r()); i += nthreads)
        tw[i] = tb.dense[i];
}

// ---- phase 1: HBM -> shared memory -------------------------------------------------
template<class F, class K>
HD void phase_load(const K k, const Pass& d, const Tables<F>& tb, const typename F::T* in,
                   typename F::T* smem, uint32_t t, uint32_t tid, uint32_t nthreads)
{
    typedef typename F::T T;
    const uint32_t R = k.lg_r(), LW = k.lg_w(), n_el = (1u << R) << LW, cs = col_stride(R);
    const uint64_t base = tile_base(t, d.in_lg_tlo, d.in_tl, d.in_th);
    const bool row_fast = k.in_row_fast();      // consecutive threads walk rows, else columns
    constexpr uint32_t EPT = 1u << F::LG_EPT;
    T v[EPT];
#pragma unroll
    for (uint32_t l = 0; l < EPT; l++) {
        uint32_t e = l * nthreads + tid;
        if (e < n_el) {
            uint32_t a = row_fast ? (e & ((1u << R) - 1)) : (e >> LW);
            uint32_t c = row_fast ? (e >> R) : (e & ((1u << LW) - 1));
            v[l] = in[base + ((uint64_t)a << d.in_lg_sa) + ((uint64_t)c << d.in_lg_sc)];
        }
    }
#pragma unroll
    for (uint32_t l = 0; l < EPT; l++) {
        uint32_t e = l * nthreads + tid;
        if (e < n_el) {
            uint32_t a = row_fast ? (e & ((1u << R) - 1)) : (e >> LW);
            uint32_t c = row_fast ? (e >> R) : (e & ((1u << LW) - 1));
            T x = F::load(v[l]);
            uint32_t nat = k.in_rev() ? brev32(a, R) : a;          // natural row index
            if (k.tw_mode() == TW_LOAD) {
                uint32_t colv = tw_column_value(d, base + ((uint64_t)c << d.in_lg_sc));
                x = F::mul(x, twiddle<F>(tb, (nat * colv) << d.tw_lsh));
            }
            smem[c * cs + swz(brev32(nat, R), c, R)] = x;            // DIT wants bit-reversed rows
        }
    }
}

// ---- phase 2: LOG_E radix-2 DIT stages on 2^LOG_E registers -----------------------
// Rows p0 + m*2^b, m < 2^LOG_E; stage t pairs m with m | (1<<t), half-size h = 2^(b+t),
// twiddle dense[h + (m mod 2^t)*2^b + j].
template<class F, class K, uint32_t LOG_E>
HD void phase_step(const K k, typename F::T* smem, uint32_t b, uint32_t tid)
{
    typedef typename F::T T;
    constexpr uint32_t E = 1u << LOG_E;
    const uint32_t R = k.lg_r(), cs = col_stride(R);
    const uint32_t lg_tpc = R >= F::LG_EPT ? R - F::LG_EPT : 0;       // threads per column
    const uint32_t c = tid >> lg_tpc, tau = tid & ((1u << lg_tpc) - 1);
    T* col = smem + c * cs;
    const T* tw = smem + (cs << k.lg_w());
    const uint32_t groups = 1u << (R - LOG_E);

    for (uint32_t g = tau; g < groups; g += (1u << lg_tpc)) {
        const uint32_t j = g & ((1u << b) - 1), hi = g >> b;
        const uint32_t p0 = (hi << (b + LOG_E)) + j;
        T x[E];
#pragma unroll
        for (uint32_t m = 0; m < E; m++)
            x[m] = col[swz(p0 + (m << b), c, R)];
#pragma unroll
        for (uint32_t t = 0; t < LOG_E; t++) {
            const uint32_t h = 1u << (b + t);
#pragma unroll
            for (uint32_t m0 = 0; m0 < E; m0++) {
                if (m0 & (1u << t)) continue;
                const uint32_t m1 = m0 | (1u << t);
                T tt;
                if (b == 0 && (m0 & ((1u << t) - 1)) == 0) {
                    // w = 1 (j = 0 when b = 0): reduce instead of multiplying by one.  The operand
                    // is loose -- a sum or difference, or at t = 0 a caller's word as loaded
                    // (F::load) -- and add/sub need a canonical second operand
                    tt = F::canon(x[m1]);
                } else {
                    const uint32_t idx = ((m0 & ((1u << t) - 1)) << b) + j;
                    tt = F::mul(x[m1], tw[h + idx]);
                }
                x[m1] = F::sub(x[m0], tt);
                x[m0] = F::add(x[m0], tt);
            }
        }
#pragma unroll
        for (uint32_t m = 0; m < E; m++)
            col[swz(p0 + (m << b), c, R)] = x[m];
    }
}

template<class F, class K>
HD void phase_step_dyn(const K k, typename F::T* smem, uint32_t b, uint32_t log_e, uint32_t tid)
{
    if constexpr (F::LG_EPT >= 4) {
        switch (log_e) {
        case 1: phase_step<F, K, 1>(k, smem, b, tid); break;
        case 2: phase_step<F, K, 2>(k, smem, b, tid); break;
        case 3: phase_step<F, K, 3>(k, smem, b, tid); break;
        default: phase_step<F, K, 4>(k, smem, b, tid); break;
        }
    } else {
        if (log_e == 1) phase_step<F, K, 1>(k, smem, b, tid);
        else phase_step<F, K, 2>(k, smem, b, tid);
    }
}

// stage schedule for a 2^R sub-NTT: full 4-stage steps first, remainder last
template<class F> HD constexpr uint32_t step_count(uint32_t R) { return (R + F::LG_EPT - 1) / F::LG_EPT; }
template<class F> HD uint32_t step_log_e(uint32_t R, uint32_t s)
{
    uint32_t done = s * F::LG_EPT;
    return R - done >= F::LG_EPT ? F::LG_EPT : R - done;
}

// ---- phase 3: shared memory -> HBM -------------------------------------------------
template<class F, class K>
HD void phase_store(const K k, const Pass& d, const Tables<F>& tb, typename F::T* out,
                    const typename F::T* smem, uint32_t t, uint32_t tid, uint32_t nthreads)
{
    typedef typename F::T T;
    const uint32_t R = k.lg_r(), LW = k.lg_w(), n_el = (1u << R) << LW, cs = col_stride(R);
    const uint64_t ibase = tile_base(t, d.in_lg_tlo, d.in_tl, d.in_th);
    const uint64_t obase = tile_base(t, d.out_lg_tlo, d.out_tl, d.out_th);
    const bool row_fast = k.out_row_fast();
    constexpr uint32_t EPT = 1u << F::LG_EPT;
#pragma unroll
    for (uint32_t l = 0; l < EPT; l++) {
        uint32_t e = l * nthreads + tid;
        if (e < n_el) {
            uint32_t v = row_fast ? (e & ((1u << R) - 1)) : (e >> LW);
            uint32_t c = row_fast ? (e >> R) : (e & ((1u << LW) - 1));
            uint32_t ka = k.out_rev() ? brev32(v, R) : v;          // natural output row
            T x = smem[c * cs + swz(ka, c, R)];
            if (k.tw_mode() == TW_STORE) {
                uint32_t colv = tw_column_value(d, ibase + ((uint64_t)c << d.in_lg_sc));
                x = F::mul(x, twiddle<F>(tb, (ka * colv) << d.tw_lsh));
            }
            if (d.scale)
                x = F::mul(x, tb.ninv);
            uint64_t row_off = (uint64_t)v << d.out_lg_sa;
            if (d.peer_on) {
                const uint32_t vl = v & ((1u << d.peer_shift) - 1);
                T* dst = reinterpret_cast<T*>(d.peer[v >> d.peer_shift]);
                dst[d.peer_block + obase + ((uint64_t)vl << d.out_lg_sa) + ((uint64_t)c << d.out_lg_sc)] = F::canon(x);
                continue;
            }
            if (d.out_split_bits)
                row_off = ((uint64_t)(v >> d.out_split_bits) << d.out_split_shift) +
                          ((uint64_t)(v & ((1u << d.out_split_bits) - 1)) << d.out_lg_sa);
            out[obase + row_off + ((uint64_t)c << d.out_lg_sc)] = F::canon(x);
        }
    }
}

// ---- matrix layout: the transforms are the columns of a row-major 2^n x width matrix ---------
// A matrix pass runs the plan of a single transform (make_plan with one transform column per
// tile, set_matrix in ntt_plan.hpp) and reads its tile columns from 2^lg_w ADJACENT matrix columns
// at one transform position: tile (t, cb) holds rows tile_base(t) + (row << lg_sa) of matrix
// columns cb * 2^lg_w + c, element (pos, col) at word pos * width + col.  Every tile row is then a
// contiguous run of 2^lg_w words, at any pass stride.  The inter-pass twiddle depends on the
// transform position only: its column is the tile's (one per tile) and the factor the row's, shared
// by all matrix columns.  Columns past `width` are masked.  The butterflies (phase_step) are the
// same; consecutive threads walk matrix columns, the strided mapping of phase_load / phase_store.
template<class F, class K>
HD void phase_load_matrix(const K k, const Pass& d, const Tables<F>& tb, const typename F::T* in,
                          typename F::T* smem, uint64_t t, uint64_t cb, uint64_t width,
                          uint32_t tid, uint32_t nthreads)
{
    typedef typename F::T T;
    const uint32_t R = k.lg_r(), LW = k.lg_w(), n_el = (1u << R) << LW, cs = col_stride(R);
    const uint64_t base = tile_base((uint32_t)t, d.in_lg_tlo, d.in_tl, d.in_th), col0 = cb << LW;
    const uint32_t colv = k.tw_mode() == TW_LOAD ? tw_column_value(d, base) : 0;
    constexpr uint32_t EPT = 1u << F::LG_EPT;
    T v[EPT];
#pragma unroll
    for (uint32_t l = 0; l < EPT; l++) {
        uint32_t e = l * nthreads + tid;
        v[l] = T{};
        if (e < n_el) {
            uint32_t a = e >> LW, c = e & ((1u << LW) - 1);
            if (col0 + c < width)
                v[l] = in[(base + ((uint64_t)a << d.in_lg_sa)) * width + col0 + c];
        }
    }
#pragma unroll
    for (uint32_t l = 0; l < EPT; l++) {
        uint32_t e = l * nthreads + tid;
        if (e < n_el) {
            uint32_t a = e >> LW, c = e & ((1u << LW) - 1);
            T x = F::load(v[l]);
            uint32_t nat = k.in_rev() ? brev32(a, R) : a;          // natural row index
            if (k.tw_mode() == TW_LOAD)
                x = F::mul(x, twiddle<F>(tb, (nat * colv) << d.tw_lsh));
            smem[c * cs + swz(brev32(nat, R), c, R)] = x;            // DIT wants bit-reversed rows
        }
    }
}

template<class F, class K>
HD void phase_store_matrix(const K k, const Pass& d, const Tables<F>& tb, typename F::T* out,
                           const typename F::T* smem, uint64_t t, uint64_t cb, uint64_t width,
                           uint32_t tid, uint32_t nthreads)
{
    typedef typename F::T T;
    const uint32_t R = k.lg_r(), LW = k.lg_w(), n_el = (1u << R) << LW, cs = col_stride(R);
    const uint64_t ibase = tile_base((uint32_t)t, d.in_lg_tlo, d.in_tl, d.in_th);
    const uint64_t obase = tile_base((uint32_t)t, d.out_lg_tlo, d.out_tl, d.out_th), col0 = cb << LW;
    const uint32_t colv = k.tw_mode() == TW_STORE ? tw_column_value(d, ibase) : 0;
    constexpr uint32_t EPT = 1u << F::LG_EPT;
#pragma unroll
    for (uint32_t l = 0; l < EPT; l++) {
        uint32_t e = l * nthreads + tid;
        if (e < n_el) {
            uint32_t v = e >> LW, c = e & ((1u << LW) - 1);
            uint32_t ka = k.out_rev() ? brev32(v, R) : v;          // natural output row
            T x = smem[c * cs + swz(ka, c, R)];
            if (k.tw_mode() == TW_STORE)
                x = F::mul(x, twiddle<F>(tb, (ka * colv) << d.tw_lsh));
            if (d.scale)
                x = F::mul(x, tb.ninv);
            if (col0 + c < width)
                out[(obase + ((uint64_t)v << d.out_lg_sa)) * width + col0 + c] = F::canon(x);
        }
    }
}

// Coset shift and LDE spread of a matrix, one row at a time (each row is one transform position,
// so one factor serves the whole row); columns c0, c0 + cstep, ... of the row.
//   coset:  row i *= g^e(i), e(i) = i, or brev(i) over lg_n bits
//   spread: output row r of 2^(lg_n + lg_blowup) = input row r >> lg_blowup times g^brev(r >> lg_blowup)
//           when the low lg_blowup bits of r are zero, zero otherwise
template<class F>
HD void coset_matrix_row(typename F::T* data, uint64_t i, uint64_t width, uint32_t lg_n, bool bitrev,
                         const typename F::T* g0, const typename F::T* g1, const typename F::T* g2,
                         uint64_t c0, uint64_t cstep)
{
    typedef typename F::T T;
    const T f = coset_mul<F>(F::one(), i, lg_n, bitrev, g0, g1, g2);
    T* row = data + i * width;
    for (uint64_t c = c0; c < width; c += cstep)
        row[c] = F::canon(F::mul(F::load(row[c]), f));
}

template<class F>
HD void lde_spread_matrix_row(typename F::T* out, const typename F::T* in, uint64_t r, uint64_t width,
                              uint32_t lg_n, uint32_t lg_blowup,
                              const typename F::T* g0, const typename F::T* g1, const typename F::T* g2,
                              uint64_t c0, uint64_t cstep)
{
    typedef typename F::T T;
    T* orow = out + r * width;
    if (r & ((1u << lg_blowup) - 1)) {
        for (uint64_t c = c0; c < width; c += cstep) orow[c] = T{};
        return;
    }
    const uint64_t i = r >> lg_blowup;
    const T f = coset_mul<F>(F::one(), i, lg_n, true, g0, g1, g2);
    const T* irow = in + i * width;
    for (uint64_t c = c0; c < width; c += cstep)
        orow[c] = F::canon(F::mul(F::load(irow[c]), f));
}

}  // namespace ntt
