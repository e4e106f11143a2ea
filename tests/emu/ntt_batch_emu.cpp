// CPU single-stepper for BATCHED NTT passes -- TEST INFRASTRUCTURE ONLY.
//
// Runs the batched descriptors (make_plan + set_batch of ntt_plan.hpp) through the exact HD phase
// functions of sppark_b200/csrc/ntt/ntt_core.cuh, tile by tile over batch x tiles, and the
// batched coset scaling through the same coset_mul the coset kernel uses.  Mirrors
// NTT::NTT_internal with batch > 1.  It is not linked into libsppark_b200.so and is not a
// fallback of any kind.
#include <vector>
#include "../../sppark_b200/csrc/ff/gl64.cuh"
#include "../../sppark_b200/csrc/ff/bb31.cuh"
#include "../../sppark_b200/csrc/ff/mont_ntt.cuh"
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
template<class F> static void coset_scale(typename F::T* data, uint32_t lg_n, size_t batch, bool bitrev, bool inverse)
{
    typedef typename F::T T;
    T g = F::group_gen();
    if (inverse) g = F::inv(g);
    std::vector<T> g0(4096), g1(4096), g2(256);
    for (uint32_t i = 0; i < 4096; i++) { g0[i] = F::pow(g, i); g1[i] = F::pow(g, (uint64_t)i << 12); }
    for (uint32_t i = 0; i < 256; i++) g2[i] = F::pow(g, (uint64_t)i << 24);
    for (size_t i = 0; i < (batch << lg_n); i++)
        data[i] = F::canon(coset_mul<F>(F::load(data[i]), i, lg_n, bitrev, g0.data(), g1.data(), g2.data()));
}

// returns the number of passes, or -1 if the plan refuses the batch term
template<class F>
static int emu_batch(typename F::T* data, uint32_t lg_n, size_t batch, int order, int inverse, int coset,
                     uint32_t lg_tile)
{
    typedef typename F::T T;
    if (lg_n == 0 || batch == 0) return 0;
    // coset exponents follow the reference's bitrev flags (NTT::NTT_internal)
    const bool in_rev = order != NN && order != NR, out_rev = order != NN && order != RN;
    if (coset && !inverse) coset_scale<F>(data, lg_n, batch, in_rev, false);
    HostTables<F> tb(lg_n, inverse != 0);
    Plan plan = make_plan(lg_n, order, inverse != 0, lg_tile, 6, F::NTT_MAX_LG_R);
    if (!set_batch(plan, batch)) return -1;
    std::vector<T> scratch(plan.needs_scratch ? batch << lg_n : 0);
    T* buf[2] = {data, scratch.data()};
    for (const Pass& d : plan.passes) {
        const uint32_t nthreads = tile_threads<F>(d);
        const uint32_t ntiles = (uint32_t)(batch << (lg_n - d.lg_r - d.lg_w));
        std::vector<T> smem(smem_elems(d));
        const KDyn k{d};
        for (uint32_t t = 0; t < ntiles; t++) {
            for (uint32_t tid = 0; tid < nthreads; tid++) phase_twiddles<F>(k, tb.view, smem.data(), tid, nthreads);
            for (uint32_t tid = 0; tid < nthreads; tid++) phase_load<F>(k, d, tb.view, buf[d.src], smem.data(), t, tid, nthreads);
            for (uint32_t s = 0; s < step_count<F>(d.lg_r); s++)
                for (uint32_t tid = 0; tid < nthreads; tid++)
                    phase_step_dyn<F>(k, smem.data(), s * F::LG_EPT, step_log_e<F>(d.lg_r, s), tid);
            for (uint32_t tid = 0; tid < nthreads; tid++) phase_store<F>(k, d, tb.view, buf[d.dst], smem.data(), t, tid, nthreads);
        }
    }
    if (coset && inverse) coset_scale<F>(data, lg_n, batch, out_rev, true);
    return (int)plan.passes.size();
}

// set_batch on a pass with slab / peer routing must refuse
extern "C" int emu_batch_rejects_slab()
{
    Plan plan = make_plan(8, NN, false, 14);
    plan.passes[0].out_split_bits = 1;
    return set_batch(plan, 2) ? 0 : 1;
}

// field ids of include/sppark_b200.h
extern "C" int emu_ntt_batch(int field, void* data, uint32_t lg_n, size_t batch, int order, int inverse, int coset,
                             uint32_t lg_tile)
{
    switch (field) {
    case 0: return emu_batch<gl64>((uint64_t*)data, lg_n, batch, order, inverse, coset, lg_tile);
    case 1: return emu_batch<bb31>((uint32_t*)data, lg_n, batch, order, inverse, coset, lg_tile);
    case 2: return emu_batch<ff::bls12_381_fr_ntt>((ff::bls12_381_fr_ntt::T*)data, lg_n, batch, order, inverse, coset, lg_tile);
    default: return -2;
    }
}
