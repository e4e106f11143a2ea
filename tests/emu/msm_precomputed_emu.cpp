// CPU single-stepper for precomputed fixed-base MSM contexts -- TEST INFRASTRUCTURE ONLY.
// Builds the table with the HD bodies of sppark_b200/csrc/msm/msm_table.cuh (in chunks, as
// msm::build_table launches them), then runs the HD pipeline bodies of msm_core.cuh over it the way
// msm_host runs a resident table: the invoked prefix cut into slices, slice s reading its points
// from row `first` of every copy, the copies N rows apart.  Not linked into the product.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <algorithm>
#include <vector>
#include "../../sppark_b200/csrc/ff/fields.cuh"
#include "../../sppark_b200/csrc/msm/msm_table.cuh"

using namespace msm;

// wbits = 0: the chooser's width (make_config_precomputed); otherwise that width
template<class F>
static Config emu_table(std::vector<uint32_t>& table, const uint32_t* points, size_t N, uint32_t wbits,
                        uint32_t copies, uint32_t chunk)
{
    constexpr uint32_t PW = 2 * F::N;
    const Config cfg = wbits ? config_for_table(N, wbits, copies, N) : make_config_precomputed(N, copies);
    table.assign((size_t)cfg.copies * N * PW, 0xdeadbeef);
    std::copy(points, points + N * PW, table.begin());
    const uint32_t K1 = cfg.copies - 1;
    std::vector<uint32_t> xyzz, zzz;
    for (size_t first = 0; K1 && first < N; first += chunk) {
        const uint32_t n = (uint32_t)std::min<size_t>(chunk, N - first), ns = n * K1;
        xyzz.assign((size_t)ns * 4 * F::N, 0xdeadbeef);
        zzz.assign((size_t)ns * F::N, 0xdeadbeef);
        for (uint32_t i = 0; i < n; i++)
            table_double_body<F>(table.data(), first, n, cfg.wbits * cfg.nwins, cfg.copies, xyzz.data(), zzz.data(), i);
        for (uint32_t tid = 0; tid * PAIR_M < ns; tid++) pair_invert_body<F>(zzz.data(), ns, tid);
        for (uint32_t s = 0; s < ns; s++) table_normalize_body<F>(xyzz.data(), zzz.data(), N, first, n, table.data(), s);
    }
    return cfg;
}

// the first m scalars against the table; info = {wbits, sets V, digits D, copies, heavy threshold}
template<class F>
static void emu_precomputed(uint32_t* out, const uint32_t* points, size_t N, const uint32_t* scalars, size_t m,
                            uint32_t wbits, uint32_t copies, uint32_t heavy, uint32_t nslices, uint32_t chunk,
                            uint32_t* info)
{
    constexpr uint32_t PW = 2 * F::N, BW = 4 * F::N, JW = 3 * F::N;
    std::vector<uint32_t> table;
    const Config tcfg = emu_table<F>(table, points, N, wbits, copies, chunk ? chunk : 1);
    // msm_resident: a one-copy context chooses its width per call, a table keeps the one it was built for
    Config cfg = tcfg.copies == 1 && !wbits ? make_config(m) : config_for_table(m, tcfg.wbits, tcfg.copies, N);
    if (heavy) { cfg.heavy = heavy; cfg.heavy_chunk = 4 * heavy; }
    const uint32_t info_[5] = {cfg.wbits, cfg.nwins, digit_count(cfg), cfg.copies, cfg.heavy};
    std::copy(info_, info_ + 5, info);
    if (m == 0) { memset(out, 0, JW * 4); return; }
    if (nslices == 0) nslices = 1;
    const size_t slice_n = (m + nslices - 1) / nslices;
    const size_t nslots = (size_t)cfg.nwins << cfg.lg_nb;
    std::vector<uint32_t> counts(nslots), offsets(nslots), cursor(nslots), sorted((size_t)cfg.nwins * cfg.copies * slice_n);
    std::vector<uint32_t> buckets(nslots * BW, 0xdeadbeef), heavy_list;
    for (size_t first = 0, sl = 0; first < m; first += slice_n, sl++) {
        // ---- one slice: msm_t::slice() with the points of rows [first, first + n) of every copy ----
        const uint32_t n = (uint32_t)std::min(slice_n, m - first);
        const uint32_t* pts = table.data() + first * PW;
        const uint32_t* sc = scalars + first * 8;
        cfg.npoints = n;
        cfg.merge = sl ? 1 : 0;
        std::fill(counts.begin(), counts.end(), 0);
        heavy_list.clear();
        for (uint32_t i = 0; i < n; i++) count_body(cfg, sc, counts.data(), i);
        for (uint32_t v = 0; v < cfg.nwins; v++) {
            uint32_t run = 0;
            for (uint32_t b = 0; b < (1u << cfg.lg_nb); b++) {
                const size_t t = ((size_t)v << cfg.lg_nb) + b;
                offsets[t] = cursor[t] = run;
                if (counts[t] > cfg.heavy) heavy_list.push_back((uint32_t)t);
                run += counts[t];
            }
        }
        for (uint32_t i = 0; i < n; i++) scatter_body(cfg, sc, cursor.data(), sorted.data(), i, 0, digit_count(cfg));
        uint32_t task_counter = 0;
        accumulate_body<F>(cfg, pts, sorted.data(), offsets.data(), counts.data(), buckets.data(), &task_counter);
        const uint32_t HT = 8;                                        // heavy kernels with 8 "threads"
        for (uint32_t t : heavy_list) {
            const uint32_t* run = sorted.data() + (size_t)(t >> cfg.lg_nb) * row_stride(cfg) + offsets[t];
            std::vector<uint32_t> tree(HT * BW);
            ec::xyzz_t<F> acc[HT];
            for (uint32_t th = 0; th < HT; th++) {
                acc[th].set_inf();
                for (uint32_t k = th; k < counts[t]; k += HT) acc[th].madd(load_point<F>(pts, run[k]));
                store_bucket<F>(tree.data(), th, acc[th]);
            }
            for (uint32_t d = HT / 2; d > 0; d >>= 1)
                for (uint32_t th = 0; th < d; th++) {
                    acc[th].add(load_bucket<F>(tree.data(), th + d));
                    store_bucket<F>(tree.data(), th, acc[th]);
                }
            if (cfg.merge) acc[0].add(load_bucket<F>(buckets.data(), t));
            store_bucket<F>(buckets.data(), t, acc[0]);
        }
    }
    const uint32_t lg_l = cfg.lg_nb > 3 ? cfg.lg_nb - 3 : 0;          // small chunks so that every level runs
    uint32_t per_win = 1u << (cfg.lg_nb - lg_l), items = cfg.nwins * per_win;
    std::vector<uint32_t> R[2], S[2];
    for (auto& v : R) v.assign((size_t)items * BW, 0);
    for (auto& v : S) v.assign((size_t)items * BW, 0);
    for (uint32_t it = 0; it < items; it++) reduce1_body<F>(cfg, buckets.data(), lg_l, R[0].data(), S[0].data(), it);
    uint32_t lg_span = lg_l, cur = 0;
    while (per_win > 1) {
        uint32_t lg_g = 31 - __builtin_clz(per_win);
        if (lg_g > 2) lg_g = 2;
        const uint32_t G = 1u << lg_g, cnt = cfg.nwins * (per_win >> lg_g);
        for (uint32_t it = 0; it < cnt; it++)
            combine_body<F>(R[cur].data(), S[cur].data(), G, lg_span, R[cur ^ 1].data(), S[cur ^ 1].data(), it);
        per_win >>= lg_g; lg_span += lg_g; cur ^= 1;
    }
    finish_body<F>(cfg, R[cur].data(), out);
}

extern "C" void emu_precomputed_bls12_381(uint32_t* out, const uint32_t* points, size_t N, const uint32_t* scalars,
                                          size_t m, uint32_t wbits, uint32_t copies, uint32_t heavy, uint32_t nslices,
                                          uint32_t chunk, uint32_t* info)
{   emu_precomputed<ff::bls12_381_fp_t>(out, points, N, scalars, m, wbits, copies, heavy, nslices, chunk, info);   }
extern "C" void emu_precomputed_pallas(uint32_t* out, const uint32_t* points, size_t N, const uint32_t* scalars,
                                       size_t m, uint32_t wbits, uint32_t copies, uint32_t heavy, uint32_t nslices,
                                       uint32_t chunk, uint32_t* info)
{   emu_precomputed<ff::pallas_fp_t>(out, points, N, scalars, m, wbits, copies, heavy, nslices, chunk, info);   }

// the chooser: copies = 0 -> make_config(n), otherwise make_config_precomputed(n, copies);
// out = {wbits, nwins, lg_nb, npoints, heavy, heavy_chunk, merge, copies, copy_stride, digits}
extern "C" void emu_config(size_t n, uint32_t copies, uint32_t* out)
{
    const Config c = copies ? make_config_precomputed(n, copies) : make_config(n);
    const uint32_t v[10] = {c.wbits, c.nwins, c.lg_nb, c.npoints, c.heavy, c.heavy_chunk, c.merge, c.copies,
                            c.copy_stride, digit_count(c)};
    std::copy(v, v + 10, out);
}
