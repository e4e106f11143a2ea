// Host-side planner: turns (lg_n, order) into the pass descriptors of ntt_core.cuh.
//
// Mirrors the role of NTT_internal / CT_NTT / GS_NTT in the reference (ntt/ntt.cuh:100-213):
// pick the algorithm from the requested input/output order and split lg_n into launches.
// Orders are the reference's InputOutputOrder {NN, NR, RN, RR} (ntt/ntt.cuh:33).
//
// Index digits: n = s_1 + ... + s_P, A_p = s_1+..+s_(p-1) bits above digit p,
// B_p = s_(p+1)+..+s_P bits below it.  See the derivations in DESIGN.md section 4.
#pragma once
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <vector>
#include "ntt_core.cuh"

namespace ntt {

// NN/NR/RN/RR are the reference's InputOutputOrder values.  In the reference RR is "GS on
// natural input, then bit_rev" (ntt/ntt.cuh:186-189,211-212): the same transform as NN, and its
// own tests assert NN == RR (poc/ntt-cuda/tests/ntt.rs:28-30).  BB is this library's extension:
// bit-reversed input AND output, in two passes without any permutation kernel.
enum Order : int { NN = 0, NR = 1, RN = 2, RR = 3, BB = 4 };

struct Plan {
    uint32_t lg_n;
    std::vector<Pass> passes;
    bool needs_scratch;
};

// lg_tile = log2 of the most elements one CTA may hold in shared memory
inline std::vector<uint32_t> split_digits(uint32_t lg_n, uint32_t max_lg_r = LG_DENSE)
{
    std::vector<uint32_t> s;
    if (const char* env = getenv("SPPARK_B200_NTT_SPLIT")) {
        // e.g. "8,8,8": honoured when it sums to lg_n (experiments / tests)
        uint32_t sum = 0;
        std::vector<uint32_t> t;
        for (const char* p = env; *p;) {
            uint32_t v = (uint32_t)strtoul(p, const_cast<char**>(&p), 10);
            if (v == 0 || v > max_lg_r) { t.clear(); break; }
            t.push_back(v);
            sum += v;
            if (*p == ',') p++;
        }
        if (!t.empty() && sum == lg_n) return t;
    }
    uint32_t P = (lg_n + max_lg_r - 1) / max_lg_r;
    if (P == 0) P = 1;
    for (uint32_t p = 0; p < P; p++)            // larger digits first
        s.push_back(lg_n / P + (p < lg_n % P ? 1 : 0));
    return s;
}

// lg_tile of the block-tile passes over `count` transforms of 2^lg_n elements side by side:
// max_lg_tile (a tile that fills one SM's shared memory), shrunk below 2^(max_lg_tile + 8) elements
// in all so that there are still >= 256 tiles for the 132 SMs.  `knob` (the value of an environment
// variable, experiments and tests) replaces the shrunk value; the result is at most max_lg_tile
inline uint32_t block_lg_tile(uint32_t lg_n, uint64_t count, uint32_t max_lg_tile, const char* knob = nullptr)
{
    uint32_t lg_total = lg_n, lg_tile = max_lg_tile;
    while (lg_total < 63 && (count >> (lg_total - lg_n)) > 1) lg_total++;   // floor(log2(count << lg_n))
    if (lg_total < lg_tile + 8) lg_tile = lg_total > 18 ? lg_total - 8 : 10;
    if (knob) lg_tile = (uint32_t)atoi(knob);
    return lg_tile > max_lg_tile ? max_lg_tile : lg_tile;
}

inline Plan make_plan(uint32_t lg_n, int order, bool inverse, uint32_t lg_tile,
                      uint32_t max_lg_w = 6, uint32_t max_lg_r = LG_DENSE)
{
    Plan plan;
    plan.lg_n = lg_n;
    const std::vector<uint32_t> s = split_digits(lg_n, max_lg_r);
    const uint32_t P = (uint32_t)s.size();
    std::vector<uint32_t> A(P), B(P);
    for (uint32_t p = 0, acc = 0; p < P; p++) { A[p] = acc; acc += s[p]; }
    for (uint32_t p = 0; p < P; p++) B[p] = lg_n - A[p] - s[p];

    if (order == RR) order = NN;
    const bool pingpong = (order == NN || order == BB) && P > 1;
    plan.needs_scratch = pingpong;
    uint32_t where = 0;                                   // buffer currently holding the data

    for (uint32_t step = 0; step < P; step++) {
        // RN runs bottom digit first, everything else top digit first
        const uint32_t p = order == RN ? P - 1 - step : step;
        const uint32_t R = s[p], a = A[p], b = B[p];
        Pass d;
        memset(&d, 0, sizeof(d));
        d.lg_r = R;

        // how many columns: fill the tile, but never wider than the digits that supply them
        uint32_t lg_w = lg_tile > R ? lg_tile - R : 0;
        if (lg_w > max_lg_w) lg_w = max_lg_w;
        uint32_t avail;                                   // bits the column index may draw from
        if (order == NR || order == RN) avail = b ? b : a;
        else if (order == NN) avail = p == 0 ? lg_n - R : (a < lg_n - R ? a : lg_n - R);
        else avail = p == P - 1 ? lg_n - R : (b < lg_n - R ? b : lg_n - R);
        if (lg_w > avail) lg_w = avail;
        d.lg_w = lg_w;
        const uint64_t W = 1ull << lg_w;

        if (order == NR || order == RN) {
            // in place: position = hi << (R+b) | row << b | low
            if (b) {
                d.in_lg_tlo = b - lg_w; d.in_tl = W; d.in_th = 1ull << (R + b);
                d.in_lg_sa = b; d.in_lg_sc = 0;
            } else {
                d.in_lg_tlo = 32; d.in_tl = W << R; d.in_th = 0;
                d.in_lg_sa = 0; d.in_lg_sc = R;
            }
            d.out_lg_tlo = d.in_lg_tlo; d.out_tl = d.in_tl; d.out_th = d.in_th;
            d.out_lg_sa = d.in_lg_sa; d.out_lg_sc = d.in_lg_sc;
            d.in_rev = order == RN; d.out_rev = order == NR;
            if (b) {
                d.tw_mode = order == NR ? TW_STORE : TW_LOAD;
                d.tw_rsh = 0; d.tw_bits = b; d.tw_brev = 0; d.tw_lsh = a;
            }
            d.src = d.dst = 0;
        } else if (order == NN) {
            // gather: position = row << (n-R) | q ; scatter: Jrest << (a+R) | k << a | Kdone
            d.in_lg_tlo = 32; d.in_tl = W; d.in_th = 0;
            d.in_lg_sa = lg_n - R; d.in_lg_sc = 0;
            if (a == 0) {
                d.out_lg_tlo = 32; d.out_tl = W << R; d.out_th = 0;
                d.out_lg_sa = 0; d.out_lg_sc = R;
            } else {
                d.out_lg_tlo = a - lg_w; d.out_tl = W; d.out_th = 1ull << (a + R);
                d.out_lg_sa = a; d.out_lg_sc = 0;
            }
            d.in_rev = 0; d.out_rev = 0;
            if (b) {
                d.tw_mode = TW_STORE; d.tw_rsh = a; d.tw_bits = b; d.tw_brev = 0; d.tw_lsh = a;
            }
        } else {
            // BB gather: position = Q << R | row ; scatter: Kdone_r << (R+b) | rk << b | Jrest_r
            d.in_lg_tlo = 32; d.in_tl = W << R; d.in_th = 0;
            d.in_lg_sa = 0; d.in_lg_sc = R;
            if (b == 0) {
                d.out_lg_tlo = 32; d.out_tl = W << R; d.out_th = 0;
                d.out_lg_sa = 0; d.out_lg_sc = R;
            } else {
                d.out_lg_tlo = b - lg_w; d.out_tl = W; d.out_th = 1ull << (R + b);
                d.out_lg_sa = b; d.out_lg_sc = 0;
            }
            d.in_rev = 1; d.out_rev = 1;
            if (b) {
                d.tw_mode = TW_STORE; d.tw_rsh = R; d.tw_bits = b; d.tw_brev = 1; d.tw_lsh = a;
            }
        }

        if (pingpong) {
            // the last pass keeps positions, so it may run in place or hop back to the caller's buffer
            d.src = where;
            d.dst = step == P - 1 ? 0 : (where ^ 1);
            where = d.dst;
        }
        d.scale = inverse && step == P - 1;
        plan.passes.push_back(d);
    }
    return plan;
}

// Turns a plan of make_plan into the same transform over `batch` rows of 2^lg_n elements stored one
// after another in every buffer the passes touch (scratch included).  The row index becomes the
// most significant digit of the tile index: a pass then has batch x its single-transform tile count,
// tile t is tile t mod 2^lg_tpt (lg_tpt = lg_n - lg_r - lg_w) of row t >> lg_tpt.  In the
// descriptor's address term th * (t >> lg_tlo) this is free: a tile layout with a high term already
// has th << (lg_tpt - lg_tlo) == 2^lg_n (the high term is the top index digit), one without
// (lg_tlo = 32) gets lg_tlo = lg_tpt, th = 2^lg_n.  Twiddle columns read bits below lg_n only
// (tw_rsh + tw_bits <= lg_n), so they see the in-row position.  No kernel changes, and batch 1
// leaves the descriptor as it is.  Slab and peer passes route rows elsewhere and cannot be batched:
// returns false for them.
inline bool set_batch(Plan& plan, uint64_t batch)
{
    for (Pass& d : plan.passes)
        if (d.out_split_bits || d.peer_on || d.tw_col_offset) return false;
    if (batch <= 1) return true;
    for (Pass& d : plan.passes) {
        const uint32_t lg_tpt = plan.lg_n - d.lg_r - d.lg_w;
        if (d.in_lg_tlo >= 32) { d.in_lg_tlo = lg_tpt; d.in_th = 1ull << plan.lg_n; }
        if (d.out_lg_tlo >= 32) { d.out_lg_tlo = lg_tpt; d.out_th = 1ull << plan.lg_n; }
    }
    return true;
}

// ---- the columns of a row-major 2^lg_n x width matrix (phase_load_matrix / phase_store_matrix) --
// Turns a plan of make_plan(lg_n, order, inverse, ., /*max_lg_w=*/0, max_lg_r) -- one transform
// column per tile, which is a complete plan of one transform -- into the same transform down every
// column of the matrix.  The transform addressing terms stay as they are; d.lg_w now counts the
// ADJACENT MATRIX COLUMNS a tile holds: as many as fill 2^lg_tile elements next to the pass's 2^lg_r
// rows, at most 2^MATRIX_MAX_LG_W, and no more than `width` needs.  A pass has 2^(lg_n - lg_r) x
// matrix_col_blocks() tiles.  Returns false for a plan with several transform columns per tile or
// with slab / peer routing.
constexpr uint32_t MATRIX_MAX_LG_W = 6;

inline bool set_matrix(Plan& plan, uint64_t width, uint32_t lg_tile)
{
    for (const Pass& d : plan.passes)
        if (d.lg_w || d.out_split_bits || d.peer_on || d.tw_col_offset) return false;
    uint32_t lg_width = 0;                                // ceil(log2(width)), capped
    while (lg_width < MATRIX_MAX_LG_W && (1ull << lg_width) < width) lg_width++;
    for (Pass& d : plan.passes) {
        const uint32_t lw = lg_tile > d.lg_r ? lg_tile - d.lg_r : 0;
        d.lg_w = lw < lg_width ? lw : lg_width;
    }
    return true;
}

inline uint64_t matrix_col_blocks(const Pass& d, uint64_t width)
{   return (width + (1ull << d.lg_w) - 1) >> d.lg_w;   }

// ---- slab-sharded transform over G = 2^lg_g ranks, ONE all-to-all ---------------------------
// N = N1 x N2 (N1 = 2^s1 rows, N2 = 2^s2 columns, x[j1*N2 + j2]).  Rank r owns the columns
// j2 in [r*N2/G, (r+1)*N2/G) of the input, stored locally as a row-major [N1][N2/G] matrix, and
// ends up owning the output coefficients X[k1 + N1*k2] with k1 in [r*N1/G, (r+1)*N1/G), stored
// as a row-major [N2][N1/G] matrix (natural order in both cases, "column slab" distribution).
//   pass 1 (local): N1-point NTT down every local column, twiddle w_N^(k1*j2) with the GLOBAL
//           column j2, written straight into the all-to-all staging layout [G][N2/G][N1/G]
//   exchange:       block q of the staging buffer goes to rank q (N*(G-1)/G^2 elements per rank)
//   after (local):  the received [N2][N1/G] matrix, N2-point NTT down every column.  N1 is the
//           first digit of the transform; when N2 exceeds one tile (lg_n > 2*max_lg_r, e.g.
//           BabyBear 2^27 = 2^9 x 2^18) the column NTT is itself the remaining digits of the
//           NN plan, run on the local array with the N1/G batch index as the finished low bits:
//           ping-pong between the received buffer and a scratch buffer, result in the former.
// The reference has no multi-GPU path; this is SURVEY.md section 8(e).
struct SlabPlan {
    uint32_t s1, s2;
    Pass pass1;
    std::vector<Pass> after;             // buffers: 0 = received matrix, 1 = scratch
    bool needs_scratch;
};

inline uint32_t slab_first_digit(uint32_t lg_n, uint32_t max_lg_r = LG_DENSE)
{
    const std::vector<uint32_t> s = split_digits(lg_n, max_lg_r);
    return s.size() < 2 ? (lg_n + 1) / 2 : s[0];
}

inline bool make_slab_plan(SlabPlan& sp, uint32_t lg_n, uint32_t lg_g, uint32_t rank, bool inverse,
                           uint32_t lg_tile, uint32_t max_lg_r = LG_DENSE, uint32_t max_lg_w = 6)
{
    std::vector<uint32_t> s = split_digits(lg_n, max_lg_r);
    if (s.size() < 2) { s.assign(2, 0); s[0] = (lg_n + 1) / 2; s[1] = lg_n - s[0]; }
    const uint32_t P = (uint32_t)s.size();
    const uint32_t s1 = s[0], s2 = lg_n - s1;
    if (s1 > max_lg_r || s1 < lg_g || s2 < lg_g) return false;
    for (uint32_t p = 1; p < P; p++)
        if (s[p] == 0 || s[p] > max_lg_r) return false;
    sp.s1 = s1;
    sp.s2 = s2;
    const uint32_t lc = s2 - lg_g;                        // log2(local columns of the input)
    const uint32_t ld = s1 - lg_g;                        // log2(local columns of the output)
    const uint32_t nloc = lg_n - lg_g;

    Pass d;
    memset(&d, 0, sizeof(d));
    d.lg_r = s1;
    uint32_t lg_w = lg_tile > s1 ? lg_tile - s1 : 0;
    if (lg_w > max_lg_w) lg_w = max_lg_w;
    if (lg_w > lc) lg_w = lc;
    d.lg_w = lg_w;
    d.in_lg_tlo = 32; d.in_tl = 1ull << lg_w; d.in_th = 0;
    d.in_lg_sa = lc; d.in_lg_sc = 0;
    d.out_lg_tlo = 32; d.out_tl = (1ull << lg_w) << ld; d.out_th = 0;
    d.out_lg_sa = 0; d.out_lg_sc = ld;
    if (lg_g) { d.out_split_bits = ld; d.out_split_shift = lc + ld; }
    d.in_rev = 0; d.out_rev = 0;
    d.tw_mode = TW_STORE; d.tw_rsh = 0; d.tw_bits = lc; d.tw_brev = 0; d.tw_lsh = 0;
    d.tw_col_offset = rank << lc;
    if (ld == 0 && lg_g) {                                // one output row per destination rank
        d.out_split_bits = 0;
        d.out_lg_sa = lc;                                 // row v == destination block v
        d.out_lg_sc = 0;
        d.out_tl = 1ull << lg_w;
    }
    d.src = 0; d.dst = 1;
    // fused-exchange variant: same tile, rows routed to the receivers (enabled by the caller
    // filling d.peer[] and setting peer_on)
    d.peer_shift = ld;                                    // ld == 0: the row IS the destination
    d.peer_block = (uint64_t)rank << (lc + ld);
    sp.pass1 = d;

    // digits 2..P on the received [N2][N1/G] array: the NN schedule of make_plan with the global
    // finished-bits count a replaced by its local value a - lg_g wherever it addresses memory
    sp.after.clear();
    sp.needs_scratch = P > 2;
    uint32_t where = 0;
    for (uint32_t p = 1, a = s1; p < P; a += s[p], p++) {
        const uint32_t R = s[p], b = lg_n - a - R, al = a - lg_g;
        memset(&d, 0, sizeof(d));
        d.lg_r = R;
        lg_w = lg_tile > R ? lg_tile - R : 0;
        if (lg_w > max_lg_w) lg_w = max_lg_w;
        const uint32_t avail = al == 0 ? nloc - R : (al < nloc - R ? al : nloc - R);
        if (lg_w > avail) lg_w = avail;
        d.lg_w = lg_w;
        const uint64_t W = 1ull << lg_w;
        d.in_lg_tlo = 32; d.in_tl = W; d.in_th = 0;
        d.in_lg_sa = nloc - R; d.in_lg_sc = 0;
        if (al == 0) {
            d.out_lg_tlo = 32; d.out_tl = W << R; d.out_th = 0;
            d.out_lg_sa = 0; d.out_lg_sc = R;
        } else {
            d.out_lg_tlo = al - lg_w; d.out_tl = W; d.out_th = 1ull << (al + R);
            d.out_lg_sa = al; d.out_lg_sc = 0;
        }
        if (b) {
            d.tw_mode = TW_STORE; d.tw_rsh = al; d.tw_bits = b; d.tw_brev = 0; d.tw_lsh = a;
        }
        if (P > 2) {
            d.src = where;
            d.dst = p == P - 1 ? 0 : (where ^ 1);
            where = d.dst;
        }
        d.scale = inverse && p == P - 1;
        sp.after.push_back(d);
    }
    return true;
}

}  // namespace ntt
