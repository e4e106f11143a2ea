// CPU single-stepper of the MSM's bucket sort -- TEST INFRASTRUCTURE ONLY.
// Executes the HD bodies of sppark_b200/csrc/msm/msm_core.cuh ("sort") in the order in which
// msm.cuh sort_slice launches its kernels; the CTA-wide steps of the bin sort (shared histogram,
// scan, placement) run as plain loops.  Not linked into the product.
#include <cstdint>
#include <cstring>
#include <algorithm>
#include <vector>
#include "../../sppark_b200/csrc/ff/fields.cuh"
#include "../../sppark_b200/csrc/msm/msm_core.cuh"

using namespace msm;

// msm_t::slice's sort (msm.cuh sort_slice), kernel by kernel; `cap` = entries per bin-sort CTA.
// ctrl / heavy_list / chunk_map in the device format (msm_core.cuh register_heavy).
struct EmuSort {
    std::vector<uint32_t> counts, offsets, cursor, sorted, ctrl, heavy_list, chunk_map;
    uint32_t lg_bins = 0, noverflow = 0;
};

static void emu_sort(const Config& cfg, const uint32_t* scalars, uint32_t cap, EmuSort& s)
{
    const uint32_t n = cfg.npoints, lg_bins = sort_lg_bins(cfg, n);
    const size_t nslots = (size_t)cfg.nwins << cfg.lg_nb, nbins = (size_t)cfg.nwins << lg_bins;
    const size_t entries = (size_t)cfg.nwins * n;
    s.lg_bins = lg_bins;
    s.counts.assign(nslots, 0);
    s.offsets.assign(nslots, 0xdeadbeef);
    s.cursor.assign(nslots, 0);
    s.sorted.assign(entries, 0xdeadbeef);
    s.ctrl.assign(4, 0);
    s.heavy_list.assign(3 * (entries / (cfg.heavy + 1) + 1), 0);
    s.chunk_map.assign(entries / cfg.heavy_chunk + entries / (cfg.heavy + 1) + 1, 0);
    std::vector<uint32_t> bin_count(nbins, 0), bin_base(nbins), bin_cur(nbins), overflow;
    std::vector<uint32_t> staging(2 * entries);
    // bin_hist_kernel
    for (uint32_t i = 0; i < n; i++)
        for_each_digit(cfg, lg_bins, scalars, i, true, cfg.nwins, [&](uint32_t, bool nz, uint32_t bin, uint32_t, uint32_t) {
            if (nz) atomic_inc(&bin_count[bin]);
        });
    // bin_scan_kernel
    for (size_t row = 0; row < nbins; row += (size_t)1 << lg_bins)
        for (uint32_t j = 0, run = 0; j < (1u << lg_bins); run += bin_count[row + j], j++)
            bin_base[row + j] = bin_cur[row + j] = run;
    // partition_kernel
    for (uint32_t i = 0; i < n; i++)
        for_each_digit(cfg, lg_bins, scalars, i, true, cfg.nwins, [&](uint32_t w, bool nz, uint32_t bin, uint32_t b, uint32_t entry) {
            if (!nz) return;
            const size_t pos = (size_t)w * n + atomic_inc(&bin_cur[bin]);
            staging[2 * pos] = entry;
            staging[2 * pos + 1] = b;
        });
    // bin_sort_kernel, one "CTA" per bin
    for (uint32_t g = 0; g < nbins; g++) {
        const uint32_t w = g >> lg_bins, bin = g & ((1u << lg_bins) - 1);
        uint32_t b0, nbk;
        if (!bin_buckets(cfg, lg_bins, w, bin, b0, nbk)) continue;
        const uint32_t cnt = bin_count[g], base = bin_base[g];
        const size_t t0 = ((size_t)w << cfg.lg_nb) + b0;
        if (last_bin(cfg, lg_bins, w, bin))
            for (uint32_t b = b0 + nbk; b < (1u << cfg.lg_nb); b++) s.offsets[((size_t)w << cfg.lg_nb) + b] = base + cnt;
        if (cnt > cap) { overflow.push_back(g); continue; }
        const uint32_t* src = staging.data() + 2 * ((size_t)w * n + base);
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
        std::copy(run.begin(), run.end(), s.sorted.begin() + (size_t)w * n + base);
    }
    // overflow_kernel<false>, overflow_scan_kernel, overflow_kernel<true>
    for (uint32_t g : overflow) {
        const uint32_t w = g >> lg_bins;
        const uint32_t* src = staging.data() + 2 * ((size_t)w * n + bin_base[g]);
        for (uint32_t k = 0; k < bin_count[g]; k++) atomic_inc(&s.counts[((size_t)w << cfg.lg_nb) + src[2 * k + 1]]);
    }
    for (uint32_t g : overflow) {
        const uint32_t w = g >> lg_bins;
        uint32_t b0, nbk;
        bin_buckets(cfg, lg_bins, w, g & ((1u << lg_bins) - 1), b0, nbk);
        const size_t t0 = ((size_t)w << cfg.lg_nb) + b0;
        for (uint32_t j = 0, acc = bin_base[g]; j < nbk; acc += s.counts[t0 + j], j++) {
            s.offsets[t0 + j] = s.cursor[t0 + j] = acc;
            register_heavy(cfg, (uint32_t)(t0 + j), s.counts[t0 + j], s.ctrl.data(), s.heavy_list.data(), s.chunk_map.data());
        }
    }
    for (uint32_t g : overflow) {
        const uint32_t w = g >> lg_bins;
        const uint32_t* src = staging.data() + 2 * ((size_t)w * n + bin_base[g]);
        for (uint32_t k = 0; k < bin_count[g]; k++)
            s.sorted[(size_t)w * n + atomic_inc(&s.cursor[((size_t)w << cfg.lg_nb) + src[2 * k + 1]])] = src[2 * k];
    }
    s.noverflow = (uint32_t)overflow.size();
}

// the sort alone (tests/test_msm_sort.py): window geometry as make_config(n) with wbits / heavy
// overridden (0 = keep), `cap` entries per bin-sort CTA.  Outputs sized by the caller: counts and
// offsets nwins << (wbits-1), sorted nwins * n, heavy one slot per heavy bucket; info =
// {nwins, heavy threshold, #heavy, lg_bins, #overflow bins}
extern "C" void emu_msm_sort(size_t n, uint32_t wbits, uint32_t heavy, uint32_t cap, const uint32_t* scalars,
                             uint32_t* counts, uint32_t* offsets, uint32_t* sorted, uint32_t* heavy_slots, uint32_t* info)
{
    Config cfg = make_config(n);
    if (wbits) { cfg.wbits = wbits; cfg.nwins = (256 + wbits - 1) / wbits; cfg.lg_nb = wbits - 1; }
    if (heavy) { cfg.heavy = heavy; cfg.heavy_chunk = 4 * heavy; }
    EmuSort st;
    emu_sort(cfg, scalars, cap, st);
    std::copy(st.counts.begin(), st.counts.end(), counts);
    std::copy(st.offsets.begin(), st.offsets.end(), offsets);
    std::copy(st.sorted.begin(), st.sorted.end(), sorted);
    for (uint32_t h = 0; h < st.ctrl[1]; h++) heavy_slots[h] = st.heavy_list[3 * h];
    const uint32_t inf[5] = {cfg.nwins, cfg.heavy, st.ctrl[1], st.lg_bins, st.noverflow};
    std::copy(inf, inf + 5, info);
}
