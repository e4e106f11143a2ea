// CPU single-stepper for MATRIX NTT passes -- TEST INFRASTRUCTURE ONLY.
//
// Runs the matrix descriptors (make_plan with one transform column per tile + set_matrix of
// ntt_plan.hpp) through the exact HD phase functions of sppark_b200/csrc/ntt/ntt_core.cuh
// (phase_load_matrix, phase_step, phase_store_matrix), tile by tile over (transform tile, column
// block), and the matrix coset shift and LDE spread through the same per-row functions the kernels
// call.  Mirrors NTTMatrix::transform and NTTMatrix::LDE_dev.  The passes whose shape has a
// statically shaped kernel in ntt.cu run with the same KShape knobs.  It is not linked into
// libsppark_b200.so and is not a fallback of any kind.
#include <vector>
#include "../../sppark_b200/csrc/ff/gl64.cuh"
#include "../../sppark_b200/csrc/ff/bb31.cuh"
#include "../../sppark_b200/csrc/ntt/ntt_plan.hpp"

using namespace ntt;

template<class F> struct HostTables {
    std::vector<typename F::T> dense, tlo, thi;
    Tables<F> view;
    HostTables(uint32_t lg_n, bool inverse)
    {
        typedef typename F::T T;
        T w_max = F::root_of_unity_max();
        if (inverse) w_max = F::inv(w_max);
        auto root = [&](uint32_t lg) {
            T w = w_max;
            for (uint32_t i = F::MAX_LG; i > lg; i--) w = F::mul(w, w);
            return w;
        };
        dense.assign(1u << LG_DENSE, F::one());
        for (uint32_t lg_h = 0; lg_h < LG_DENSE; lg_h++) {
            uint32_t h = 1u << lg_h;
            T w = root(lg_h + 1), acc = F::one();
            for (uint32_t i = 0; i < h; i++, acc = F::mul(acc, w)) dense[h + i] = acc;
        }
        T wn = root(lg_n);
        tlo.resize(1u << LG_TLO);
        T acc = F::one();
        for (uint32_t i = 0; i < (1u << LG_TLO); i++, acc = F::mul(acc, wn)) tlo[i] = acc;
        uint32_t nhi = lg_n > LG_TLO ? 1u << (lg_n - LG_TLO) : 1;
        thi.resize(nhi);
        T step = acc;
        acc = F::one();
        for (uint32_t i = 0; i < nhi; i++, acc = F::mul(acc, step)) thi[i] = acc;
        T half = F::inv(F::add(F::one(), F::one()));
        T ninv = F::one();
        for (uint32_t i = 0; i < lg_n; i++) ninv = F::mul(ninv, half);
        view = Tables<F>{dense.data(), tlo.data(), thi.data(), ninv};
    }
};

// g^i, g^(i << 12), g^(i << 24) (g^-1 for inverse transforms), as gen_coset_kernel builds them
template<class F> struct CosetTables {
    std::vector<typename F::T> g0, g1, g2;
    explicit CosetTables(bool inverse) : g0(4096), g1(4096), g2(256)
    {
        typename F::T g = F::group_gen();
        if (inverse) g = F::inv(g);
        for (uint32_t i = 0; i < 4096; i++) { g0[i] = F::pow(g, i); g1[i] = F::pow(g, (uint64_t)i << 12); }
        for (uint32_t i = 0; i < 256; i++) g2[i] = F::pow(g, (uint64_t)i << 24);
    }
};

template<class F, class K>
static void run_pass(const Pass& d, const Tables<F>& tb, const typename F::T* in, typename F::T* out,
                     uint64_t width, uint32_t lg_n)
{
    const K k{d};
    const uint32_t nthreads = tile_threads<F>(d);
    const uint64_t ncb = matrix_col_blocks(d, width), nt = 1ull << (lg_n - d.lg_r);
    std::vector<typename F::T> smem(smem_elems(d));
    for (uint64_t i = 0; i < nt * ncb; i++) {                // the kernel's tile order: i = t * ncb + cb
        const uint64_t t = i / ncb, cb = i % ncb;
        for (uint32_t tid = 0; tid < nthreads; tid++) phase_twiddles<F>(k, tb, smem.data(), tid, nthreads);
        for (uint32_t tid = 0; tid < nthreads; tid++)
            phase_load_matrix<F>(k, d, tb, in, smem.data(), t, cb, width, tid, nthreads);
        for (uint32_t s = 0; s < step_count<F>(d.lg_r); s++)
            for (uint32_t tid = 0; tid < nthreads; tid++)
                phase_step_dyn<F>(k, smem.data(), s * F::LG_EPT, step_log_e<F>(d.lg_r, s), tid);
        for (uint32_t tid = 0; tid < nthreads; tid++)
            phase_store_matrix<F>(k, d, tb, out, smem.data(), t, cb, width, tid, nthreads);
    }
}

// the shapes with a statically shaped kernel in ntt.cu (launch_matrix) run with its knobs
template<class F, uint32_t R, uint32_t W>
static bool try_shape(const Pass& d, const Tables<F>& tb, const typename F::T* in, typename F::T* out,
                      uint64_t width, uint32_t lg_n)
{
    if (d.lg_r != R || d.lg_w != W) return false;
    run_pass<F, KShape<R, W>>(d, tb, in, out, width, lg_n);
    return true;
}

// returns the number of passes, -1 if set_matrix refuses the plan
template<class F>
static int emu_matrix(typename F::T* data, uint32_t lg_n, uint64_t width, int order, int inverse, int coset,
                      uint32_t lg_tile)
{
    typedef typename F::T T;
    if (lg_n == 0 || width == 0) return 0;
    const bool in_rev = order != NN && order != NR, out_rev = order != NN && order != RN;
    const uint64_t rows = 1ull << lg_n;
    if (coset && !inverse) {
        CosetTables<F> ct(false);
        for (uint64_t r = 0; r < rows; r++)
            coset_matrix_row<F>(data, r, width, lg_n, in_rev, ct.g0.data(), ct.g1.data(), ct.g2.data(), 0, 1);
    }
    HostTables<F> tb(lg_n, inverse != 0);
    Plan plan = make_plan(lg_n, order, inverse != 0, lg_tile, 0, F::NTT_MAX_LG_R);
    if (!set_matrix(plan, width, lg_tile)) return -1;
    std::vector<T> scratch(plan.needs_scratch ? width << lg_n : 0);
    T* buf[2] = {data, scratch.data()};
    for (const Pass& d : plan.passes) {
        if (!(try_shape<F, 12, 2>(d, tb.view, buf[d.src], buf[d.dst], width, lg_n)
              || try_shape<F, 11, 3>(d, tb.view, buf[d.src], buf[d.dst], width, lg_n)
              || try_shape<F, 10, 4>(d, tb.view, buf[d.src], buf[d.dst], width, lg_n)
              || try_shape<F, 10, 3>(d, tb.view, buf[d.src], buf[d.dst], width, lg_n)
              || try_shape<F, 8, 4>(d, tb.view, buf[d.src], buf[d.dst], width, lg_n)))
            run_pass<F, KDyn>(d, tb.view, buf[d.src], buf[d.dst], width, lg_n);
    }
    if (coset && inverse) {
        CosetTables<F> ct(true);
        for (uint64_t r = 0; r < rows; r++)
            coset_matrix_row<F>(data, r, width, lg_n, out_rev, ct.g0.data(), ct.g1.data(), ct.g2.data(), 0, 1);
    }
    return (int)plan.passes.size();
}

// NTTMatrix::LDE_dev: inverse NR on d_in, the spread with the coset shift, forward RN on d_out.  The
// spread walks each row's columns with a stride of 3 from three starting columns, as a block's
// threads do
template<class F>
static int emu_lde(typename F::T* out, typename F::T* in, uint32_t lg_n, uint32_t lg_blowup, uint64_t width,
                   uint32_t lg_tile)
{
    if (emu_matrix<F>(in, lg_n, width, NR, 1, 0, lg_tile) < 0) return -1;
    CosetTables<F> ct(false);
    for (uint64_t r = 0; r < (1ull << (lg_n + lg_blowup)); r++)
        for (uint64_t c0 = 0; c0 < 3; c0++)
            lde_spread_matrix_row<F>(out, in, r, width, lg_n, lg_blowup, ct.g0.data(), ct.g1.data(), ct.g2.data(), c0, 3);
    return emu_matrix<F>(out, lg_n + lg_blowup, width, RN, 0, 0, lg_tile);
}

// set_matrix on a plan with several transform columns per tile, or slab / peer routing, must refuse
extern "C" int emu_matrix_rejects()
{
    Plan wide = make_plan(16, NN, false, 14);                 // 8 + 8, max_lg_w = 6: 2^6 columns per tile
    Plan slab = make_plan(8, NN, false, 14, 0);
    slab.passes[0].out_split_bits = 1;
    return !set_matrix(wide, 4, 14) && !set_matrix(slab, 4, 14) ? 1 : 0;
}

// (lg_r, lg_w) of pass p of the matrix plan, -1 past the last pass
extern "C" int emu_matrix_shape(uint32_t lg_n, uint64_t width, int order, uint32_t lg_tile, uint32_t p)
{
    Plan plan = make_plan(lg_n, order, false, lg_tile, 0, 12);
    if (!set_matrix(plan, width, lg_tile) || p >= plan.passes.size()) return -1;
    return (int)(plan.passes[p].lg_r << 8 | plan.passes[p].lg_w);
}

// field ids of include/sppark_b200.h
extern "C" int emu_ntt_matrix(int field, void* data, uint32_t lg_n, uint64_t width, int order, int inverse, int coset,
                              uint32_t lg_tile)
{
    switch (field) {
    case 0: return emu_matrix<gl64>((uint64_t*)data, lg_n, width, order, inverse, coset, lg_tile);
    case 1: return emu_matrix<bb31>((uint32_t*)data, lg_n, width, order, inverse, coset, lg_tile);
    default: return -2;
    }
}

extern "C" int emu_lde_matrix(int field, void* out, void* in, uint32_t lg_n, uint32_t lg_blowup, uint64_t width,
                              uint32_t lg_tile)
{
    switch (field) {
    case 0: return emu_lde<gl64>((uint64_t*)out, (uint64_t*)in, lg_n, lg_blowup, width, lg_tile);
    case 1: return emu_lde<bb31>((uint32_t*)out, (uint32_t*)in, lg_n, lg_blowup, width, lg_tile);
    default: return -2;
    }
}
