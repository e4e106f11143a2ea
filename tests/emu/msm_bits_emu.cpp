// CPU single-stepper for the MSM pipeline over small scalars -- TEST INFRASTRUCTURE ONLY.
// Executes the HD kernel bodies of sppark_b200/csrc/msm/msm_core.cuh (portable arithmetic branch)
// in the order msm_t launches them, for a Config built by make_config(n, nbits, scalar_bytes):
// count / scatter read scalar_bytes per scalar and walk ceil((nbits + 1) / c) digits.  The same
// sequence as tests/emu/msm_emu.cpp without the batched-affine variant.  Not linked into the product.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <algorithm>
#include <vector>
#include "../../sppark_b200/csrc/ff/fields.cuh"
#include "../../sppark_b200/csrc/msm/msm_core.cuh"

using namespace msm;

// wbits 0: the chooser's width; heavy 0: the chooser's threshold; the points in nslices slices that
// share one bucket file (the host-pointer pipeline)
template<class F>
static void emu_msm_bits(uint32_t* out, const uint32_t* points_all, size_t npoints_all, const uint32_t* scalars_all,
                         uint32_t scalar_bytes, uint32_t nbits, uint32_t wbits, uint32_t heavy, uint32_t nslices)
{
    constexpr uint32_t BW = 4 * F::N, JW = 3 * F::N;
    if (npoints_all == 0) { memset(out, 0, JW * 4); return; }
    Config cfg = make_config(npoints_all, nbits, scalar_bytes);
    if (wbits) { cfg.wbits = wbits; cfg.nwins = digits_for(nbits, wbits); cfg.lg_nb = wbits - 1; }
    if (heavy) { cfg.heavy = heavy; cfg.heavy_chunk = 4 * heavy; }
    const size_t nslots = (size_t)cfg.nwins << cfg.lg_nb;
    std::vector<uint32_t> counts(nslots), offsets(nslots), cursor(nslots), sorted((size_t)cfg.nwins * npoints_all);
    std::vector<uint32_t> buckets(nslots * BW, 0xdeadbeef), heavy_list;
    if (nslices == 0) nslices = 1;
    const size_t slice_n = (npoints_all + nslices - 1) / nslices;
    for (size_t first = 0, sl = 0; first < npoints_all; first += slice_n, sl++) {
        const size_t npoints = std::min(slice_n, npoints_all - first);
        const uint32_t* points = points_all + first * 2 * F::N;
        const uint32_t* scalars = scalars_all + first * (scalar_bytes / 4);
        cfg.npoints = (uint32_t)npoints;
        cfg.merge = sl ? 1 : 0;
        std::fill(counts.begin(), counts.end(), 0);
        heavy_list.clear();
        for (uint32_t i = 0; i < npoints; i++) count_body(cfg, scalars, counts.data(), i);
        for (uint32_t w = 0; w < cfg.nwins; w++) {
            uint32_t run = 0;
            for (uint32_t b = 0; b < (1u << cfg.lg_nb); b++) {
                const size_t t = ((size_t)w << cfg.lg_nb) + b;
                offsets[t] = cursor[t] = run;
                if (counts[t] > cfg.heavy) heavy_list.push_back((uint32_t)t);
                run += counts[t];
            }
        }
        for (uint32_t i = 0; i < npoints; i++) scatter_body(cfg, scalars, cursor.data(), sorted.data(), i, 0, cfg.nwins);
        uint32_t task_counter = 0;
        accumulate_body<F>(cfg, points, sorted.data(), offsets.data(), counts.data(), buckets.data(), &task_counter);
        for (uint32_t t : heavy_list) {                              // heavy kernels, one "thread" per bucket
            const uint32_t* run = sorted.data() + (size_t)(t >> cfg.lg_nb) * cfg.npoints + offsets[t];
            ec::xyzz_t<F> acc;
            acc.set_inf();
            for (uint32_t k = 0; k < counts[t]; k++) acc.madd(load_point<F>(points, run[k]));
            if (cfg.merge) acc.add(load_bucket<F>(buckets.data(), t));
            store_bucket<F>(buckets.data(), t, acc);
        }
    }
    const uint32_t lg_l = cfg.lg_nb > 3 ? cfg.lg_nb - 3 : 0;         // small chunks so that every level runs
    uint32_t per_win = 1u << (cfg.lg_nb - lg_l), items = cfg.nwins * per_win;
    std::vector<uint32_t> R[2], S[2];
    for (auto& v : R) v.assign((size_t)items * BW, 0);
    for (auto& v : S) v.assign((size_t)items * BW, 0);
    for (uint32_t it = 0; it < items; it++) reduce1_body<F>(cfg, buckets.data(), lg_l, R[0].data(), S[0].data(), it);
    uint32_t lg_span = lg_l, cur = 0;
    while (per_win > 1) {
        uint32_t lg_g = 31 - __builtin_clz(per_win);
        if (lg_g > 2) lg_g = 2;
        const uint32_t G = 1u << lg_g, n = cfg.nwins * (per_win >> lg_g);
        for (uint32_t it = 0; it < n; it++)
            combine_body<F>(R[cur].data(), S[cur].data(), G, lg_span, R[cur ^ 1].data(), S[cur ^ 1].data(), it);
        per_win >>= lg_g; lg_span += lg_g; cur ^= 1;
    }
    finish_body<F>(cfg, R[cur].data(), out);
}

extern "C" void emu_msm_bls12_381_bits(uint32_t* out, const uint32_t* points, size_t n, const uint32_t* scalars,
                                       uint32_t scalar_bytes, uint32_t nbits, uint32_t wbits, uint32_t heavy,
                                       uint32_t nslices)
{   emu_msm_bits<ff::bls12_381_fp_t>(out, points, n, scalars, scalar_bytes, nbits, wbits, heavy, nslices);   }
