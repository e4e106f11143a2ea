// CPU single-stepper for batched MSMs (Config::nvecs > 1) -- TEST INFRASTRUCTURE ONLY.
// B scalar vectors against one point set, in groups of G vectors: per group the HD bodies of
// sppark_b200/csrc/msm/msm_core.cuh run in the order msm_t launches them -- the bin sort (bin histogram
// over groups of `wpg` windows as bin_hist_kernel walks them, partition, bin sort with the overflow
// path for bins past `cap`), accumulate, heavy buckets, reduce / combine and one finish per vector --
// over the G V bucket sets of the group.  Tables are built by the bodies of msm_table.cuh, as in
// tests/emu/msm_precomputed_emu.cpp.  Not linked into the product.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <algorithm>
#include <vector>
#include "../../sppark_b200/csrc/ff/fields.cuh"
#include "../../sppark_b200/csrc/msm/msm_table.cuh"

using namespace msm;

// the sort of one group (msm.cuh sort_slice_sw), kernel by kernel
struct EmuSort {
    std::vector<uint32_t> counts, offsets, cursor, sorted, ctrl, heavy_list, chunk_map;
    uint32_t noverflow = 0;
};

template<uint32_t SW>
static void emu_sort(const Config& cfg, const uint32_t* scalars, uint32_t cap, uint32_t wpg, EmuSort& s)
{
    const uint32_t n = cfg.npoints, lg_bins = sort_lg_bins(cfg, row_stride(cfg)), V = vec_sets(cfg);
    const size_t rs = row_stride(cfg);
    const size_t nslots = (size_t)cfg.nwins << cfg.lg_nb, nbins = (size_t)cfg.nwins << lg_bins;
    const size_t entries = (size_t)cfg.nwins * rs;
    s.counts.assign(nslots, 0);
    s.offsets.assign(nslots, 0xdeadbeef);
    s.cursor.assign(nslots, 0);
    s.sorted.assign(entries, 0xdeadbeef);
    s.ctrl.assign(4, 0);
    s.heavy_list.assign(3 * (entries / (cfg.heavy + 1) + 1), 0);
    s.chunk_map.assign(entries / cfg.heavy_chunk + entries / (cfg.heavy + 1) + 1, 0);
    std::vector<uint32_t> bin_count(nbins, 0), bin_base(nbins), bin_cur(nbins), overflow;
    std::vector<uint32_t> staging(2 * entries);
    // bin_hist_kernel: window groups [w0, w0 + wpg), the vectors whose sets meet them
    const uint32_t D = digit_count(cfg);
    for (uint32_t w0 = 0; w0 < cfg.nwins; w0 += wpg) {
        const uint32_t w1 = std::min(w0 + wpg, cfg.nwins);
        for (uint32_t g = w0 / V; g * V < w1; g++) {
            const uint32_t d_end = cfg.copies > 1 ? D : std::min(D, w1 - g * V);
            for (uint32_t i = 0; i < n; i++)
                for_each_digit<SW>(cfg, lg_bins, scalars, i, true, d_end, [&](uint32_t w, bool nz, uint32_t bin, uint32_t, uint32_t) {
                    if (w >= w0 && w < w1 && nz) atomic_inc(&bin_count[bin]);
                }, g);
        }
    }
    // bin_scan_kernel
    for (size_t row = 0; row < nbins; row += (size_t)1 << lg_bins)
        for (uint32_t j = 0, run = 0; j < (1u << lg_bins); run += bin_count[row + j], j++)
            bin_base[row + j] = bin_cur[row + j] = run;
    // partition_kernel
    for (uint32_t g = 0; g < cfg.nvecs; g++)
        for (uint32_t i = 0; i < n; i++)
            for_each_digit<SW>(cfg, lg_bins, scalars, i, true, D, [&](uint32_t w, bool nz, uint32_t bin, uint32_t b, uint32_t entry) {
                if (!nz) return;
                const size_t pos = (size_t)w * rs + atomic_inc(&bin_cur[bin]);
                staging[2 * pos] = entry;
                staging[2 * pos + 1] = b;
            }, g);
    // bin_sort_kernel, one "CTA" per bin
    for (uint32_t gb = 0; gb < nbins; gb++) {
        const uint32_t w = gb >> lg_bins, bin = gb & ((1u << lg_bins) - 1);
        uint32_t b0, nbk;
        if (!bin_buckets(cfg, lg_bins, w, bin, b0, nbk)) continue;
        const uint32_t cnt = bin_count[gb], base = bin_base[gb];
        const size_t t0 = ((size_t)w << cfg.lg_nb) + b0;
        if (last_bin(cfg, lg_bins, w, bin))
            for (uint32_t b = b0 + nbk; b < (1u << cfg.lg_nb); b++) s.offsets[((size_t)w << cfg.lg_nb) + b] = base + cnt;
        if (cnt > cap) { overflow.push_back(gb); continue; }
        const uint32_t* src = staging.data() + 2 * ((size_t)w * rs + base);
        std::vector<uint32_t> cur(nbk, 0), run(cnt);
        for (uint32_t k = 0; k < cnt; k++) atomic_inc(&cur[src[2 * k + 1] - b0]);
        for (uint32_t j = 0, acc = 0; j < nbk; j++) {
            const uint32_t c = cur[j];
            s.counts[t0 + j] = c;
            s.offsets[t0 + j] = base + acc;
            cur[j] = acc;
            register_heavy(cfg, (uint32_t)(t0 + j), c, s.ctrl.data(), s.heavy_list.data(), s.chunk_map.data());
            acc += c;
        }
        for (uint32_t k = 0; k < cnt; k++) run[atomic_inc(&cur[src[2 * k + 1] - b0])] = src[2 * k];
        std::copy(run.begin(), run.end(), s.sorted.begin() + (size_t)w * rs + base);
    }
    // overflow_kernel<false>, overflow_scan_kernel, overflow_kernel<true>
    for (uint32_t gb : overflow) {
        const uint32_t w = gb >> lg_bins;
        const uint32_t* src = staging.data() + 2 * ((size_t)w * rs + bin_base[gb]);
        for (uint32_t k = 0; k < bin_count[gb]; k++) atomic_inc(&s.counts[((size_t)w << cfg.lg_nb) + src[2 * k + 1]]);
    }
    for (uint32_t gb : overflow) {
        const uint32_t w = gb >> lg_bins;
        uint32_t b0, nbk;
        bin_buckets(cfg, lg_bins, w, gb & ((1u << lg_bins) - 1), b0, nbk);
        const size_t t0 = ((size_t)w << cfg.lg_nb) + b0;
        for (uint32_t j = 0, acc = bin_base[gb]; j < nbk; acc += s.counts[t0 + j], j++) {
            s.offsets[t0 + j] = s.cursor[t0 + j] = acc;
            register_heavy(cfg, (uint32_t)(t0 + j), s.counts[t0 + j], s.ctrl.data(), s.heavy_list.data(), s.chunk_map.data());
        }
    }
    for (uint32_t gb : overflow) {
        const uint32_t w = gb >> lg_bins;
        const uint32_t* src = staging.data() + 2 * ((size_t)w * rs + bin_base[gb]);
        for (uint32_t k = 0; k < bin_count[gb]; k++)
            s.sorted[(size_t)w * rs + atomic_inc(&s.cursor[((size_t)w << cfg.lg_nb) + src[2 * k + 1]])] = src[2 * k];
    }
    s.noverflow = (uint32_t)overflow.size();
}

// one group: sort -> accumulate -> heavy -> reduce / combine -> one finish per vector (out: G points)
template<class F>
static void emu_group(const Config& cfg, const uint32_t* pts, const uint32_t* scalars, uint32_t cap, uint32_t wpg,
                      uint32_t* out, uint32_t* stats)
{
    constexpr uint32_t BW = 4 * F::N, JW = 3 * F::N;
    EmuSort s;
    switch (cfg.swords) {
    case 1: emu_sort<1>(cfg, scalars, cap, wpg, s); break;
    case 2: emu_sort<2>(cfg, scalars, cap, wpg, s); break;
    case 4: emu_sort<4>(cfg, scalars, cap, wpg, s); break;
    default: emu_sort<8>(cfg, scalars, cap, wpg, s); break;
    }
    const size_t nslots = (size_t)cfg.nwins << cfg.lg_nb;
    std::vector<uint32_t> buckets(nslots * BW, 0xdeadbeef);
    uint32_t task_counter = 0;
    accumulate_body<F>(cfg, pts, s.sorted.data(), s.offsets.data(), s.counts.data(), buckets.data(), &task_counter);
    for (uint32_t h = 0; h < s.ctrl[1]; h++) {                       // heavy buckets, one "CTA" each
        const uint32_t t = s.heavy_list[3 * h];
        const uint32_t* run = s.sorted.data() + (size_t)(t >> cfg.lg_nb) * row_stride(cfg) + s.offsets[t];
        ec::xyzz_t<F> acc;
        acc.set_inf();
        for (uint32_t k = 0; k < s.counts[t]; k++) acc.madd(load_point<F>(pts, run[k]));
        store_bucket<F>(buckets.data(), t, acc);
    }
    stats[0] += s.ctrl[1];
    stats[1] += s.noverflow;
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
    const uint32_t V = vec_sets(cfg);
    for (uint32_t b = 0; b < cfg.nvecs; b++)                          // finish_par_kernel: CTA b
        finish_body<F>(cfg, R[cur].data() + (size_t)b * V * BW, out + (size_t)b * JW);
}

// batch vectors of n <= N scalars (scalar_bytes each, bits from nbits up ignored) against the first n of
// N points.  copies 0 / 1: plain points, width wbits (0: make_config's); copies > 1: a table of up to that
// many copies, width wbits (0: make_config_precomputed's).  group: vectors per group (0: all).  heavy: the
// threshold (0: the chooser's); cap: entries per bin-sort CTA; wpg: windows per histogram group.
// info = {wbits, V, digits, copies, heavy threshold, groups, #heavy buckets, #overflow bins}
template<class F>
static void emu_batch(uint32_t* out, const uint32_t* points, size_t N, const uint32_t* scalars, size_t n,
                      size_t batch, uint32_t group, uint32_t scalar_bytes, uint32_t nbits, uint32_t wbits,
                      uint32_t copies, uint32_t heavy, uint32_t cap, uint32_t wpg, uint32_t* info)
{
    constexpr uint32_t PW = 2 * F::N, JW = 3 * F::N;
    std::vector<uint32_t> table(points, points + N * PW);
    Config cfg1;
    if (copies > 1) {
        const Config tcfg = wbits ? config_for_table(N, wbits, copies, N) : make_config_precomputed(N, copies);
        table.resize((size_t)tcfg.copies * N * PW);
        const uint32_t K1 = tcfg.copies - 1, ns = (uint32_t)N * K1;
        std::vector<uint32_t> xyzz((size_t)ns * 4 * F::N), zzz((size_t)ns * F::N);
        for (uint32_t i = 0; K1 && i < N; i++)
            table_double_body<F>(table.data(), 0, (uint32_t)N, tcfg.wbits * tcfg.nwins, tcfg.copies, xyzz.data(), zzz.data(), i);
        for (uint32_t tid = 0; K1 && tid * PAIR_M < ns; tid++) pair_invert_body<F>(zzz.data(), ns, tid);
        for (uint32_t sl = 0; K1 && sl < ns; sl++)
            table_normalize_body<F>(xyzz.data(), zzz.data(), N, 0, (uint32_t)N, table.data(), sl);
        cfg1 = config_for_table(n, tcfg.wbits, tcfg.copies, N, nbits, scalar_bytes);
    } else {
        cfg1 = wbits ? config_for_table(n, wbits, 1, N, nbits, scalar_bytes) : make_config(n, nbits, scalar_bytes);
    }
    if (heavy) { cfg1.heavy = heavy; cfg1.heavy_chunk = 4 * heavy; }
    const size_t G = group ? group : batch;
    uint32_t stats[2] = {0, 0}, ngroups = 0;
    if (n == 0) memset(out, 0, batch * JW * 4);
    for (size_t v0 = 0; n && v0 < batch; v0 += G, ngroups++) {
        const Config cfg = group_config(cfg1, (uint32_t)std::min(G, batch - v0));
        emu_group<F>(cfg, table.data(), scalars + v0 * n * (scalar_bytes / 4), cap ? cap : 24576, wpg ? wpg : cfg.nwins,
                     out + v0 * JW, stats);
    }
    const uint32_t v[8] = {cfg1.wbits, cfg1.nwins, digit_count(cfg1), cfg1.copies, cfg1.heavy, ngroups, stats[0], stats[1]};
    std::copy(v, v + 8, info);
}

#define EMU_BATCH(name, F)                                                                                           \
extern "C" void emu_batch_##name(uint32_t* out, const uint32_t* points, size_t N, const uint32_t* scalars, size_t n,  \
                                 size_t batch, uint32_t group, uint32_t scalar_bytes, uint32_t nbits, uint32_t wbits,  \
                                 uint32_t copies, uint32_t heavy, uint32_t cap, uint32_t wpg, uint32_t* info)        \
{   emu_batch<F>(out, points, N, scalars, n, batch, group, scalar_bytes, nbits, wbits, copies, heavy, cap, wpg, info);   }
EMU_BATCH(bls12_381, ff::bls12_381_fp_t)
EMU_BATCH(pallas, ff::pallas_fp_t)
