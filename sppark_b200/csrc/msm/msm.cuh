// msm_t<Curve>: device-side Pippenger driver (the role of the reference's msm_t,
// msm/pippenger.cuh:325-747).  Kernels are thin __global__ wrappers over msm_core.cuh.
#pragma once
#include "../util/gpu.cuh"
#include "msm_core.cuh"
#include "msm_pair.cuh"
#include "msm_table.cuh"
#include "msm_scale.cuh"

namespace msm {

#ifndef SPPARK_B200_ACC_THREADS
# define SPPARK_B200_ACC_THREADS 128
#endif
#ifndef SPPARK_B200_ACC_MIN_BLOCKS
# define SPPARK_B200_ACC_MIN_BLOCKS 3
#endif
constexpr uint32_t ACC_THREADS = SPPARK_B200_ACC_THREADS;       // accumulate CTA size
constexpr uint32_t HEAVY_THREADS = 128;

// ---- sort (msm_core.cuh, "sort"): bin histogram -> bin scan -> partition -> bin sort -> overflow ----
constexpr uint32_t HIST_THREADS = 1024;
constexpr uint32_t HIST_SMEM_WORDS = 56 * 1024;     // bin counters of one histogram CTA (224 KB)
constexpr uint32_t SORT_THREADS = 512;
// entries one bin-sort CTA places through shared memory: with the 2^SORT_SMAX bucket cursors 112 KB,
// two CTAs per SM.  Uniform windows fill a bin to ~2^13 entries at any size up to 2^28 points; the
// top window of 254-bit scalars fills its used bins to ~2^14.
constexpr uint32_t SORT_CAP = 24576;

// exclusive prefix over len values (four consecutive per thread, tiles of 4 * blockDim);
// visit(j, value_j, prefix_j) for every j < len, returns the total.  Every thread of the CTA calls it.
template<class Load, class Visit>
__device__ uint32_t block_exclusive_scan(uint32_t len, Load load, Visit visit)
{
    __shared__ uint32_t warp_tot[32];
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
    uint32_t carry = 0;                                             // total of the tiles before this one
    for (uint32_t t0 = 0; t0 < len; t0 += 4 * blockDim.x) {
        const uint32_t b = t0 + 4 * threadIdx.x;
        uint32_t c[4];
#pragma unroll
        for (uint32_t k = 0; k < 4; k++) c[k] = b + k < len ? load(b + k) : 0;
        const uint32_t s = c[0] + c[1] + c[2] + c[3];
        uint32_t x = s;                                             // inclusive scan inside the warp
#pragma unroll
        for (uint32_t d = 1; d < 32; d <<= 1) {
            const uint32_t y = __shfl_up_sync(0xffffffffu, x, d);
            if (lane >= d) x += y;
        }
        if (lane == 31) warp_tot[wid] = x;
        __syncthreads();
        if (wid == 0) {
            uint32_t t = lane < nw ? warp_tot[lane] : 0;
#pragma unroll
            for (uint32_t d = 1; d < 32; d <<= 1) {
                const uint32_t y = __shfl_up_sync(0xffffffffu, t, d);
                if (lane >= d) t += y;
            }
            warp_tot[lane] = t;
        }
        __syncthreads();
        uint32_t r = carry + (wid ? warp_tot[wid - 1] : 0) + x - s;
        carry += warp_tot[31];
#pragma unroll
        for (uint32_t k = 0; k < 4; k++) {
            if (b + k < len) visit(b + k, c[k], r);
            r += c[k];
        }
        __syncthreads();                                            // warp_tot is reused by the next tile
    }
    return carry;
}

// pass 1: bin histogram of the windows [w0, w0 + wpg) of group blockIdx.y in shared memory, one
// global atomic per non-zero counter per CTA; a warp adds equal bins once (all scalars equal:
// every lane of the warp hits one counter).  With a table every digit is walked: its set is w mod V.
// A batch walks the vectors whose sets meet [w0, w1).
// One instantiation per scalar width SW (cfg.swords words), each scalar read with one load of its width.
template<uint32_t SW>
__global__ void __launch_bounds__(HIST_THREADS)
bin_hist_kernel(const Config cfg, uint32_t lg_bins, const uint32_t* scalars, uint32_t wpg, uint32_t* bin_count)
{
    extern __shared__ uint32_t hist[];
    const uint32_t w0 = blockIdx.y * wpg, w1 = min(w0 + wpg, cfg.nwins), nctr = (w1 - w0) << lg_bins;
    const uint32_t V = vec_sets(cfg), D = digit_count(cfg);
    const uint32_t lane = threadIdx.x & 31;
    for (uint32_t k = threadIdx.x; k < nctr; k += blockDim.x) hist[k] = 0;
    __syncthreads();
    for (uint32_t g = w0 / V; g * V < w1; g++) {
        // without a table digit w of vector g lands in set gV + w: the digits of sets past w1 are not walked
        const uint32_t d_end = cfg.copies > 1 ? D : min(D, w1 - g * V);
        for (uint32_t i0 = blockIdx.x * blockDim.x + (threadIdx.x & ~31u); i0 < cfg.npoints; i0 += gridDim.x * blockDim.x) {
            const uint32_t i = i0 + lane;                           // whole warps iterate together
            for_each_digit<SW>(cfg, lg_bins, scalars, i, i < cfg.npoints, d_end,
                           [&](uint32_t w, bool nz, uint32_t bin, uint32_t, uint32_t) {
                if (w < w0 || w >= w1) return;                      // the same for the whole warp
                const uint32_t key = nz ? bin - (w0 << lg_bins) : ~0u;
                const uint32_t peers = __match_any_sync(0xffffffffu, key);
                if (nz && lane == __ffs(peers) - 1) atomicAdd(&hist[key], __popc(peers));
            }, g);
        }
    }
    __syncthreads();
    for (uint32_t k = threadIdx.x; k < nctr; k += blockDim.x)
        if (hist[k]) atomicAdd(&bin_count[((size_t)w0 << lg_bins) + k], hist[k]);
}

// one CTA per window: window-local bin bases, and the partition's cursors
static __global__ void __launch_bounds__(1024)
bin_scan_kernel(uint32_t lg_bins, const uint32_t* bin_count, uint32_t* bin_base, uint32_t* bin_cur)
{
    const size_t row = (size_t)blockIdx.x << lg_bins;
    block_exclusive_scan(1u << lg_bins, [&](uint32_t j) { return bin_count[row + j]; },
                         [&](uint32_t j, uint32_t, uint32_t off) { bin_base[row + j] = off; bin_cur[row + j] = off; });
}

// pass 2: every (point, window) entry appended at its bin's cursor, one reservation per distinct
// bin per warp.  All windows in one pass: the open frontier is one partly written line per bin
// (nwins * 2^lg_bins * 128 B, 13.6 MB at 2^26 points; a batch's group is sized to keep it under
// BATCH_FRONTIER), so lines fill in L2 and leave whole.  A batch's vectors one after the other.
template<uint32_t SW>
__global__ void __launch_bounds__(256)
partition_kernel(const Config cfg, uint32_t lg_bins, const uint32_t* scalars, uint32_t* bin_cur, uint2* staging)
{
    const uint32_t lane = threadIdx.x & 31;
    for (uint32_t g = 0; g < cfg.nvecs; g++)
        for (uint32_t i0 = blockIdx.x * blockDim.x + (threadIdx.x & ~31u); i0 < cfg.npoints; i0 += gridDim.x * blockDim.x) {
            const uint32_t i = i0 + lane;
            for_each_digit<SW>(cfg, lg_bins, scalars, i, i < cfg.npoints, digit_count(cfg),
                           [&](uint32_t w, bool nz, uint32_t bin, uint32_t b, uint32_t entry) {
                const uint32_t peers = __match_any_sync(0xffffffffu, nz ? bin : ~0u);
                const uint32_t leader = __ffs(peers) - 1;
                uint32_t pos = 0;
                if (nz && lane == leader) pos = atomicAdd(&bin_cur[bin], __popc(peers));
                pos = __shfl_sync(0xffffffffu, pos, leader) + __popc(peers & ((1u << lane) - 1));
                if (nz) staging[(size_t)w * row_stride(cfg) + pos] = make_uint2(entry, b);
            }, g);
        }
}

// pass 3: one CTA per bin (blockIdx.x = w << lg_bins | bin).  Bucket histogram of the bin in
// shared memory, counts / offsets / heavy buckets for its buckets, the entries placed into a
// shared copy of the bin's output range, which is then written out coalesced.  A bin of more than
// `cap` entries is listed for the overflow path instead.
static __global__ void __launch_bounds__(SORT_THREADS)
bin_sort_kernel(const Config cfg, uint32_t lg_bins, uint32_t cap, const uint2* staging, const uint32_t* bin_count,
                const uint32_t* bin_base, uint32_t* counts, uint32_t* offsets, uint32_t* sorted, uint32_t* ctrl,
                uint32_t* heavy_list, uint32_t* chunk_map, uint32_t* overflow)
{
    extern __shared__ uint32_t sm[];                        // [cap] output run, [2^SORT_SMAX] bucket cursors
    const uint32_t w = blockIdx.x >> lg_bins, bin = blockIdx.x & ((1u << lg_bins) - 1);
    uint32_t b0, nbk;
    if (!bin_buckets(cfg, lg_bins, w, bin, b0, nbk)) return;
    const uint32_t cnt = bin_count[blockIdx.x], base = bin_base[blockIdx.x];
    const size_t t0 = ((size_t)w << cfg.lg_nb) + b0;
    if (last_bin(cfg, lg_bins, w, bin))                     // buckets no digit reaches (top window)
        for (uint32_t b = b0 + nbk + threadIdx.x; b < (1u << cfg.lg_nb); b += blockDim.x)
            offsets[((size_t)w << cfg.lg_nb) + b] = base + cnt;
    if (cnt > cap) {
        if (threadIdx.x == 0) overflow[atomicAdd(&ctrl[3], 1)] = blockIdx.x;
        return;
    }
    uint32_t *run = sm, *cur = sm + cap;
    for (uint32_t k = threadIdx.x; k < nbk; k += blockDim.x) cur[k] = 0;
    __syncthreads();
    const uint2* src = staging + (size_t)w * row_stride(cfg) + base;
    for (uint32_t k = threadIdx.x; k < cnt; k += blockDim.x) atomicAdd(&cur[src[k].y - b0], 1);
    __syncthreads();
    block_exclusive_scan(nbk, [&](uint32_t j) { return cur[j]; }, [&](uint32_t j, uint32_t c, uint32_t off) {
        counts[t0 + j] = c;
        offsets[t0 + j] = base + off;
        cur[j] = off;
        register_heavy(cfg, (uint32_t)(t0 + j), c, ctrl, heavy_list, chunk_map);
    });
    for (uint32_t k = threadIdx.x; k < cnt; k += blockDim.x) {
        const uint2 e = src[k];
        run[atomicAdd(&cur[e.y - b0], 1)] = e.x;
    }
    __syncthreads();
    uint32_t* dst = sorted + (size_t)w * row_stride(cfg) + base;
    for (uint32_t k = threadIdx.x; k < cnt; k += blockDim.x) dst[k] = run[k];
}

// overflow path, over the entries of every listed bin in turn (grid-stride): PLACE = false adds
// them to `slots` = counts, PLACE = true places them at `slots` = cursor.  One global atomic per
// distinct bucket per warp: a bucket holding every point costs n / 32 atomics.
template<bool PLACE>
__global__ void __launch_bounds__(256)
overflow_kernel(const Config cfg, uint32_t lg_bins, const uint2* staging, const uint32_t* bin_count,
                const uint32_t* bin_base, const uint32_t* ctrl, const uint32_t* overflow, uint32_t* slots,
                uint32_t* sorted)
{
    const uint32_t lane = threadIdx.x & 31, nov = ctrl[3];
    for (uint32_t o = 0; o < nov; o++) {
        const uint32_t g = overflow[o], w = g >> lg_bins, cnt = bin_count[g];
        const uint2* src = staging + (size_t)w * row_stride(cfg) + bin_base[g];
        uint32_t* row = slots + ((size_t)w << cfg.lg_nb);
        for (uint32_t k0 = blockIdx.x * blockDim.x + (threadIdx.x & ~31u); k0 < cnt; k0 += gridDim.x * blockDim.x) {
            const uint32_t k = k0 + lane;
            const uint2 e = k < cnt ? src[k] : make_uint2(0, ~0u);
            const uint32_t peers = __match_any_sync(0xffffffffu, e.y);
            const uint32_t leader = __ffs(peers) - 1;
            uint32_t pos = 0;
            if (k < cnt && lane == leader) pos = atomicAdd(&row[e.y], __popc(peers));
            if (PLACE) {
                pos = __shfl_sync(0xffffffffu, pos, leader) + __popc(peers & ((1u << lane) - 1));
                if (k < cnt) sorted[(size_t)w * row_stride(cfg) + pos] = e.x;
            }
        }
    }
}

// overflow path, between the two passes: one CTA per listed bin, offsets / cursors / heavy buckets
static __global__ void __launch_bounds__(1024)
overflow_scan_kernel(const Config cfg, uint32_t lg_bins, const uint32_t* bin_base, const uint32_t* overflow,
                     const uint32_t* counts, uint32_t* offsets, uint32_t* cursor, uint32_t* ctrl,
                     uint32_t* heavy_list, uint32_t* chunk_map)
{
    const uint32_t nov = ctrl[3];
    for (uint32_t o = blockIdx.x; o < nov; o += gridDim.x) {
        const uint32_t g = overflow[o], w = g >> lg_bins, base = bin_base[g];
        uint32_t b0, nbk;
        bin_buckets(cfg, lg_bins, w, g & ((1u << lg_bins) - 1), b0, nbk);
        const size_t t0 = ((size_t)w << cfg.lg_nb) + b0;
        block_exclusive_scan(nbk, [&](uint32_t j) { return counts[t0 + j]; }, [&](uint32_t j, uint32_t c, uint32_t off) {
            offsets[t0 + j] = base + off;
            cursor[t0 + j] = base + off;
            register_heavy(cfg, (uint32_t)(t0 + j), c, ctrl, heavy_list, chunk_map);
        });
    }
}

// device buffers of the sort; nbins = nwins << sort_lg_bins(cfg, slice capacity).
// control block ctrl: [0] accumulate's task counter, [1] #heavy buckets, [2] #chunks, [3] #overflow bins
struct SortBufs {
    uint32_t *counts, *offsets, *cursor, *ctrl, *heavy_list, *chunk_map, *sorted;
    uint32_t *bin_count, *bin_base, *bin_cur, *overflow;
    uint2* staging;                 // nwins * slice capacity entries
};

// finer profile marks inside the sort (tools/probe_msm_sort.py); off by default, so that the
// "sort" phase stays one number
inline bool sort_profile() { const char* e = getenv("SPPARK_B200_MSM_SORT_PROFILE"); return e && atoi(e) != 0; }

// (window, bucket) lists of cfg.npoints scalars: counts, offsets, sorted, ctrl[1..3], heavy_list,
// chunk_map.  cap <= SORT_CAP: entries per bin-sort CTA (smaller values send more bins down the
// overflow path; the self-test uses that).  SW = cfg.swords: the scalar width of d_scalars.
template<uint32_t SW>
void sort_slice_sw(const Config& cfg, uint32_t cap, const uint32_t* d_scalars, const SortBufs& s, uint32_t sms,
                   cudaStream_t stream)
{
    const uint32_t lg_bins = sort_lg_bins(cfg, row_stride(cfg));
    const size_t nbins = (size_t)cfg.nwins << lg_bins, nslots = (size_t)cfg.nwins << cfg.lg_nb;
    const bool marks = sort_profile();
    CUDA_OK(cudaFuncSetAttribute(bin_hist_kernel<SW>, cudaFuncAttributeMaxDynamicSharedMemorySize, HIST_SMEM_WORDS * 4));
    CUDA_OK(cudaFuncSetAttribute(bin_sort_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (SORT_CAP + (1u << SORT_SMAX)) * 4));
    CUDA_OK(cudaMemsetAsync(s.counts, 0, nslots * 4, stream));
    CUDA_OK(cudaMemsetAsync(s.ctrl, 0, 16, stream));
    CUDA_OK(cudaMemsetAsync(s.bin_count, 0, nbins * 4, stream));
    const uint32_t wpg = std::min(cfg.nwins, HIST_SMEM_WORDS >> lg_bins);
    const uint32_t ngroups = (cfg.nwins + wpg - 1) / wpg;
    const uint32_t hist_blk = (uint32_t)std::min<size_t>((cfg.npoints + HIST_THREADS - 1) / HIST_THREADS, sms);
    bin_hist_kernel<SW><<<dim3(hist_blk, ngroups), HIST_THREADS, ((size_t)wpg << lg_bins) * 4, stream>>>(
        cfg, lg_bins, d_scalars, wpg, s.bin_count);
    COUNT_LAUNCH();
    bin_scan_kernel<<<cfg.nwins, 1024, 0, stream>>>(lg_bins, s.bin_count, s.bin_base, s.bin_cur);
    COUNT_LAUNCH();
    if (marks) g_profile.mark("sort_partition", stream);
    const uint32_t part_blk = (uint32_t)std::min<size_t>((cfg.npoints + 255) / 256, (size_t)sms * 8);
    partition_kernel<SW><<<part_blk, 256, 0, stream>>>(cfg, lg_bins, d_scalars, s.bin_cur, s.staging);
    COUNT_LAUNCH();
    if (marks) g_profile.mark("sort_bins", stream);
    bin_sort_kernel<<<(uint32_t)nbins, SORT_THREADS, (cap + (1u << SORT_SMAX)) * 4, stream>>>(
        cfg, lg_bins, cap, s.staging, s.bin_count, s.bin_base, s.counts, s.offsets, s.sorted, s.ctrl,
        s.heavy_list, s.chunk_map, s.overflow);
    COUNT_LAUNCH();
    if (marks) g_profile.mark("sort_overflow", stream);
    overflow_kernel<false><<<sms * 4, 256, 0, stream>>>(cfg, lg_bins, s.staging, s.bin_count, s.bin_base, s.ctrl,
                                                        s.overflow, s.counts, s.sorted);
    overflow_scan_kernel<<<sms, 1024, 0, stream>>>(cfg, lg_bins, s.bin_base, s.overflow, s.counts, s.offsets, s.cursor,
                                                   s.ctrl, s.heavy_list, s.chunk_map);
    overflow_kernel<true><<<sms * 4, 256, 0, stream>>>(cfg, lg_bins, s.staging, s.bin_count, s.bin_base, s.ctrl,
                                                       s.overflow, s.cursor, s.sorted);
    COUNT_LAUNCH(); COUNT_LAUNCH(); COUNT_LAUNCH();
    CUDA_OK(cudaGetLastError());
}

inline void sort_slice(const Config& cfg, uint32_t cap, const uint32_t* d_scalars, const SortBufs& s, uint32_t sms,
                       cudaStream_t stream)
{
    switch (cfg.swords) {
    case 1: sort_slice_sw<1>(cfg, cap, d_scalars, s, sms, stream); break;
    case 2: sort_slice_sw<2>(cfg, cap, d_scalars, s, sms, stream); break;
    case 4: sort_slice_sw<4>(cfg, cap, d_scalars, s, sms, stream); break;
    case 8: sort_slice_sw<8>(cfg, cap, d_scalars, s, sms, stream); break;
    default: throw cuda_error(-(int)cudaErrorInvalidValue, "msm: scalars must be 4, 8, 16 or 32 bytes");
    }
}

// ---- batched-affine pre-reduction of the bucket lists (msm_pair.cuh) ---------------------------
static __global__ void pair_counts_kernel(const Config cfg, const uint32_t* counts, uint32_t* counts1, uint32_t nslots)
{
    for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < nslots; t += gridDim.x * blockDim.x)
        pair_counts_body(cfg, counts, counts1, t);
}

// one CTA (1024 threads) per window: window-local exclusive prefix of counts1, window total
static __global__ void __launch_bounds__(1024)
pair_scan_kernel(const Config cfg, const uint32_t* counts1, uint32_t* off1, uint32_t* wintotal)
{
    __shared__ uint32_t warp_tot[32];
    const uint32_t w = blockIdx.x, nb = 1u << cfg.lg_nb, lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const size_t base = (size_t)w << cfg.lg_nb;
    uint32_t carry = 0;
    for (uint32_t t0 = 0; t0 < nb; t0 += 4096) {
        const uint32_t b = t0 + threadIdx.x * 4;
        uint4 c = make_uint4(0, 0, 0, 0);
        if (b < nb) c = *reinterpret_cast<const uint4*>(counts1 + base + b);
        const uint32_t s = c.x + c.y + c.z + c.w;
        uint32_t x = s;
#pragma unroll
        for (uint32_t d = 1; d < 32; d <<= 1) {
            uint32_t y = __shfl_up_sync(0xffffffffu, x, d);
            if (lane >= d) x += y;
        }
        if (lane == 31) warp_tot[wid] = x;
        __syncthreads();
        if (wid == 0) {
            uint32_t t = warp_tot[lane];
#pragma unroll
            for (uint32_t d = 1; d < 32; d <<= 1) {
                uint32_t y = __shfl_up_sync(0xffffffffu, t, d);
                if (lane >= d) t += y;
            }
            warp_tot[lane] = t;
        }
        __syncthreads();
        uint4 r;
        r.x = carry + (wid ? warp_tot[wid - 1] : 0) + x - s;
        r.y = r.x + c.x;
        r.z = r.y + c.y;
        r.w = r.z + c.z;
        carry += warp_tot[31];
        if (b < nb) *reinterpret_cast<uint4*>(off1 + base + b) = r;
        __syncthreads();
    }
    if (threadIdx.x == 0) wintotal[w] = carry;
}

static __global__ void pair_winbase_kernel(const Config cfg, const uint32_t* wintotal, uint32_t* winbase)
{
    if (blockIdx.x || threadIdx.x) return;
    uint32_t run = 0;
    for (uint32_t w = 0; w < cfg.nwins; w++) { winbase[w] = run; run += wintotal[w]; }
    winbase[cfg.nwins] = run;
}

template<class F>
__global__ void __launch_bounds__(128)
pair_forward_kernel(const Config cfg, const uint32_t* points, const uint32_t* sorted, const uint32_t* offsets,
                    const uint32_t* counts, const uint32_t* counts1, const uint32_t* off1, const uint32_t* winbase,
                    uint32_t o0, uint32_t nthreads, uint32_t* pre, uint32_t* totals)
{
    const uint32_t tid = blockIdx.x * blockDim.x + threadIdx.x;
    if (tid < nthreads)
        pair_forward_body<F>(cfg, points, sorted, offsets, counts, counts1, off1, winbase, o0, nthreads, pre, totals, tid);
}

template<class F>
__global__ void __launch_bounds__(128)
pair_invert_kernel(uint32_t* totals, uint32_t n)
{
    pair_invert_body<F>(totals, n, blockIdx.x * blockDim.x + threadIdx.x);
}

template<class F>
__global__ void __launch_bounds__(128)
pair_backward_kernel(const Config cfg, const uint32_t* points, const uint32_t* sorted, const uint32_t* offsets,
                     const uint32_t* counts, const uint32_t* counts1, const uint32_t* off1, const uint32_t* winbase,
                     uint32_t o0, uint32_t nthreads, const uint32_t* pre, const uint32_t* totals_inv, uint32_t* out)
{
    const uint32_t tid = blockIdx.x * blockDim.x + threadIdx.x;
    if (tid < nthreads)
        pair_backward_body<F>(cfg, points, sorted, offsets, counts, counts1, off1, winbase, o0, nthreads, pre,
                              totals_inv, out, tid);
}

template<class F>
__global__ void __launch_bounds__(ACC_THREADS, (F::N > 12 ? 2 : SPPARK_B200_ACC_MIN_BLOCKS))
accumulate_direct_kernel(const Config cfg, const uint32_t* sums, const uint32_t* offsets, const uint32_t* counts,
                         uint32_t* buckets, uint32_t* task_counter, const uint32_t* counts1, const uint32_t* off1,
                         const uint32_t* winbase)
{
    accumulate_body<F, true>(cfg, sums, nullptr, offsets, counts, buckets, task_counter, counts1, off1, winbase);
}

template<class F>
__global__ void __launch_bounds__(ACC_THREADS, (F::N > 12 ? 2 : SPPARK_B200_ACC_MIN_BLOCKS))
accumulate_kernel(const Config cfg, const uint32_t* points, const uint32_t* sorted,
                  const uint32_t* offsets, const uint32_t* counts, uint32_t* buckets,
                  uint32_t* task_counter)
{
    accumulate_body<F>(cfg, points, sorted, offsets, counts, buckets, task_counter);
}

// block-wide sum of one xyzz per thread through shared memory; result valid in thread 0
template<class F>
DEV void block_sum(ec::xyzz_t<F>& acc, uint32_t* tree)
{
    store_bucket<F>(tree, threadIdx.x, acc);
    __syncthreads();
    for (uint32_t d = blockDim.x / 2; d > 0; d >>= 1) {
        if (threadIdx.x < d) {
            acc.add_hot(load_bucket<F>(tree, threadIdx.x + d));
            store_bucket<F>(tree, threadIdx.x, acc);
        }
        __syncthreads();
    }
}

// heavy buckets, phase A: one CTA per cfg.heavy_chunk entries -> one partial sum per chunk, so a
// bucket holding most of the points is spread over the whole GPU
template<class F>
__global__ void __launch_bounds__(HEAVY_THREADS)
heavy_chunks_kernel(const Config cfg, const uint32_t* points, const uint32_t* sorted,
                    const uint32_t* offsets, const uint32_t* counts, const uint32_t* ctrl,
                    const uint32_t* heavy_list, const uint32_t* chunk_map, uint32_t* partials)
{
    extern __shared__ __align__(16) uint32_t tree[];         // HEAVY_THREADS xyzz slots
    const uint32_t nchunks = ctrl[2];
    for (uint32_t ch = blockIdx.x; ch < nchunks; ch += gridDim.x) {
        const uint32_t h = chunk_map[ch], t = heavy_list[3 * h], k0 = (ch - heavy_list[3 * h + 1]) * cfg.heavy_chunk;
        const uint32_t cnt = counts[t], k1 = min(k0 + cfg.heavy_chunk, cnt);
        const uint32_t* run = sorted + (size_t)(t >> cfg.lg_nb) * row_stride(cfg) + offsets[t];
        ec::xyzz_t<F> acc;
        acc.set_inf();
        for (uint32_t k = k0 + threadIdx.x; k < k1; k += blockDim.x)
            acc.madd(load_point<F>(points, run[k]));
        block_sum<F>(acc, tree);
        if (threadIdx.x == 0) store_bucket<F>(partials, ch, acc);
        __syncthreads();
    }
}

// phase B: one CTA per heavy bucket folds that bucket's chunk partials
template<class F>
__global__ void __launch_bounds__(HEAVY_THREADS)
heavy_fold_kernel(const Config cfg, const uint32_t* ctrl, const uint32_t* heavy_list,
                  const uint32_t* partials, uint32_t* buckets)
{
    extern __shared__ __align__(16) uint32_t tree[];
    const uint32_t nheavy = ctrl[1];
    for (uint32_t h = blockIdx.x; h < nheavy; h += gridDim.x) {
        const uint32_t t = heavy_list[3 * h], first = heavy_list[3 * h + 1], nch = heavy_list[3 * h + 2];
        ec::xyzz_t<F> acc;
        acc.set_inf();
        for (uint32_t k = threadIdx.x; k < nch; k += blockDim.x)
            acc.add_hot(load_bucket<F>(partials, first + k));
        block_sum<F>(acc, tree);
        if (threadIdx.x == 0) {
            if (cfg.merge) acc.add_hot(load_bucket<F>(buckets, t));
            store_bucket<F>(buckets, t, acc);
        }
        __syncthreads();
    }
}

// 3 CTAs/SM: the <= 4096 items per window of a 2^26 MSM (416 CTAs) then fit one wave of 444
// resident CTAs; at 255 registers (2 CTAs/SM) they took two
template<class F>
__global__ void __launch_bounds__(128, (F::N > 12 ? 2 : 3))
reduce1_kernel(const Config cfg, const uint32_t* buckets, uint32_t lg_l, uint32_t nitems,
               uint32_t* outR, uint32_t* outS)
{
    uint32_t item = blockIdx.x * blockDim.x + threadIdx.x;
    if (item < nitems) reduce1_body<F>(cfg, buckets, lg_l, outR, outS, item);
}

template<class F>
__global__ void __launch_bounds__(128)
combine_kernel(const uint32_t* inR, const uint32_t* inS, uint32_t G, uint32_t lg_span,
               uint32_t nitems, uint32_t* outR, uint32_t* outS)
{
    uint32_t item = blockIdx.x * blockDim.x + threadIdx.x;
    if (item < nitems) combine_body<F>(inR, inS, G, lg_span, outR, outS, item);
}

template<class F>
__global__ void finish_kernel(const Config cfg, const uint32_t* winR, uint32_t* out)
{
    if (blockIdx.x == 0 && threadIdx.x == 0) finish_body<F>(cfg, winR, out);
}

// ---- finish on four lanes -------------------------------------------------------------------------
// The Horner combination of the window sums is one dependent chain of nwins*c doublings; what can
// run side by side are the multiplications INSIDE a point operation: a doubling (dbl-2008-s-1) is
// three rounds of independent products {V = U^2, Q = X^2}, {W = UV, S = XV, M^2}, {M(S-X3), WY,
// ZZ*V, ZZZ*W}, a full addition four.  Lanes 0..3 of one warp execute the shared ladder in
// lock-step on different operands (one instruction stream, SIMD), values travel through a few
// shared-memory slots: 3 ladder latencies per doubling instead of 9, 4 per addition instead of
// 14 (the same group element as finish_body, which the CPU single-stepper keeps running).
template<class F> struct Par4 {
    enum { sX, sY, sZZZ, sZZ, sA, sB, sC, sD, sE, sF, sG, sH, NS };
    // slot i of the accumulator: its four coordinates first, then eight scratch values that
    // several accumulators of one lane group may share
    struct Slots {
        F* pt;
        F* tmp;
        __device__ F& operator[](uint32_t i) const { return i < 4 ? pt[i] : tmp[i - 4]; }
    };
    Slots s;
    uint32_t lane;
    unsigned mask;                                          // the four lanes of this group
    __device__ Par4(F* pt, F* tmp, uint32_t lane_, unsigned mask_ = 0xFu) : s{pt, tmp}, lane(lane_), mask(mask_) {}
    __device__ void sync() const { __syncwarp(mask); }
    __device__ ec::xyzz_t<F> get() const
    {
        ec::xyzz_t<F> p;
        p.X = s[sX]; p.Y = s[sY]; p.ZZZ = s[sZZZ]; p.ZZ = s[sZZ];
        return p;
    }
    __device__ void set_inf()
    {
        if (lane == 0) { s[sX] = F::zero(); s[sY] = F::zero(); s[sZZZ] = F::zero(); s[sZZ] = F::zero(); }
        sync();
    }
    __device__ bool is_inf() const { return s[sZZZ].is_zero() && s[sZZ].is_zero(); }

    // lane-wise choice of an operand: every lane then makes THE SAME call of the shared ladder (one
    // instruction stream for the four products; a branch per lane would serialise them)
    __device__ F pick(const F& a0, const F& a1, const F& a2, const F& a3) const
    {
        F r;
#pragma unroll
        for (int i = 0; i < F::N; i++)
            r.l[i] = lane == 0 ? a0.l[i] : lane == 1 ? a1.l[i] : lane == 2 ? a2.l[i] : a3.l[i];
        return r;
    }
    __device__ void put(uint32_t i0, uint32_t i1, uint32_t i2, uint32_t i3, const F& r)
    {   s[lane == 0 ? i0 : lane == 1 ? i1 : lane == 2 ? i2 : i3] = r;   }

    __device__ void dbl()
    {
        if (is_inf()) return;                               // same decision on all four lanes
        const F U = s[sY].dbl(), X = s[sX];
        F r = F::mul_shared(pick(U, X, X, X), pick(U, X, X, X));
        put(sA, sB, sB, sB, r);                             // sA = V = U^2, sB = Q = X^2
        sync();
        const F V = s[sA];
        F M = s[sB];
        M = M.dbl() + M;
        r = F::mul_shared(pick(U, X, M, M), pick(V, V, M, M));
        put(sC, sD, sE, sE, r);                             // sC = W, sD = S, sE = M^2
        sync();
        const F W = s[sC], S = s[sD];
        const F X3 = s[sE] - S - S;
        const F Y = s[sY], ZZ = s[sZZ], ZZZ = s[sZZZ];
        sync();                                             // everyone has read the old point
        r = F::mul_shared(pick(M, W, ZZ, ZZZ), pick(S - X3, Y, V, W));
        put(sF, sG, sZZ, sZZZ, r);
        sync();
        if (lane == 0) { s[sY] = s[sF] - s[sG]; s[sX] = X3; }
        sync();
    }

    // point += p2 (both XYZZ); p2 in registers of every lane
    __device__ void add(const ec::xyzz_t<F>& p2)
    {
        if (p2.is_inf()) return;
        if (is_inf()) {
            if (lane == 0) { s[sX] = p2.X; s[sY] = p2.Y; s[sZZZ] = p2.ZZZ; s[sZZ] = p2.ZZ; }
            sync();
            return;
        }
        const F X1 = s[sX], Y1 = s[sY], ZZZ1 = s[sZZZ], ZZ1 = s[sZZ];
        F r = F::mul_shared(pick(X1, Y1, p2.X, p2.Y), pick(p2.ZZ, p2.ZZZ, ZZ1, ZZZ1));
        put(sA, sB, sC, sD, r);                             // sA = U1, sB = S1, sC = U2, sD = S2
        sync();
        const F U1 = s[sA], S1 = s[sB];
        const F P = s[sC] - U1, R = s[sD] - S1;
        sync();
        if (P.is_zero()) {                                  // same decision on all four lanes
            if (R.is_zero()) dbl();
            else { if (lane == 0) { s[sZZZ] = F::zero(); s[sZZ] = F::zero(); } sync(); }
            return;
        }
        r = F::mul_shared(pick(P, R, ZZ1, ZZZ1), pick(P, R, p2.ZZ, p2.ZZZ));
        put(sE, sF, sG, sH, r);                             // sE = PP, sF = RR, sG = ZZ1*ZZ2, sH = ZZZ1*ZZZ2
        sync();
        const F PP = s[sE], G = s[sG];
        r = F::mul_shared(pick(P, U1, G, G), PP);
        put(sA, sC, sZZ, sZZ, r);                           // sA = PPP, sC = Q, ZZ3
        sync();
        const F PPP = s[sA], Q = s[sC], H = s[sH];
        const F X3 = s[sF] - PPP - Q - Q;
        r = F::mul_shared(pick(R, S1, H, H), pick(Q - X3, PPP, PPP, PPP));
        put(sD, sE, sZZZ, sZZZ, r);                         // T1, T2, ZZZ3
        sync();
        if (lane == 0) { s[sY] = s[sD] - s[sE]; s[sX] = X3; }
        sync();
    }
};

// combine level (see combine_body) with four lanes per item: the chains of a level are G x 3 full
// additions long and there are only a few thousand items, so latency, not throughput, sets its
// time; the additions run as four rounds of lane-parallel products
// four-lane groups per CTA: 20 field elements of shared memory each (30 KB for 48-byte Fp at 32
// groups; Fp2 elements are twice as wide, so half as many groups)
template<class F> struct par_groups { static constexpr uint32_t value = F::N <= 12 ? 32 : 16; };

template<class F>
__global__ void __launch_bounds__(4 * par_groups<F>::value)
combine_par_kernel(const uint32_t* inR, const uint32_t* inS, uint32_t G, uint32_t lg_span,
                   uint32_t nitems, uint32_t* outR, uint32_t* outS)
{
    __shared__ F sm[par_groups<F>::value][20];                   // per group: acc, weighted, rsum, 8 scratch
    const uint32_t grp = threadIdx.x >> 2, lane = threadIdx.x & 3;
    const uint32_t item = blockIdx.x * par_groups<F>::value + grp;
    if (item >= nitems) return;                             // whole groups leave together
    const unsigned mask = 0xFu << ((threadIdx.x & 31) & ~3u);
    F* base = sm[grp];
    Par4<F> acc(base, base + 12, lane, mask), weighted(base + 4, base + 12, lane, mask), rsum(base + 8, base + 12, lane, mask);
    acc.set_inf();
    weighted.set_inf();
    rsum.set_inf();
    const size_t first = (size_t)item * G;
    for (uint32_t i = G; i-- > 0;) {
        rsum.add(load_bucket<F>(inR, first + i));
        acc.add(load_bucket<F>(inS, first + i));
        if (i) weighted.add(acc.get());                     // sum_{i>=1} i*S_i
    }
    for (uint32_t d = 0; d < lg_span; d++) weighted.dbl();
    rsum.add(weighted.get());
    if (lane == 0) {
        store_bucket<F>(outR, item, rsum.get());
        store_bucket<F>(outS, item, acc.get());
    }
}

// one CTA per vector of the group: CTA b folds the V window sums of sets [bV, bV + V) into the
// Jacobian point b of out_jacobian
template<class F>
__global__ void __launch_bounds__(32)
finish_par_kernel(const Config cfg, const uint32_t* winR, uint32_t* out_jacobian)
{
    __shared__ F slots[Par4<F>::NS];
    if (threadIdx.x >= 4) return;
    const uint32_t V = vec_sets(cfg);
    winR += (size_t)blockIdx.x * V * 4 * F::N;
    out_jacobian += (size_t)blockIdx.x * 3 * F::N;
    Par4<F> p(slots, slots + 4, threadIdx.x);
    {
        const ec::xyzz_t<F> top = load_bucket<F>(winR, V - 1);
        if (p.lane == 0) { slots[Par4<F>::sX] = top.X; slots[Par4<F>::sY] = top.Y; slots[Par4<F>::sZZZ] = top.ZZZ; slots[Par4<F>::sZZ] = top.ZZ; }
        p.sync();
    }
    for (uint32_t w = V - 1; w-- > 0;) {
        for (uint32_t d = 0; d < cfg.wbits; d++) p.dbl();
        p.add(load_bucket<F>(winR, w));
    }
    // XYZZ -> Jacobian (X*ZZ, Y*ZZZ, ZZ), canonical limbs; infinity -> all zero
    const bool inf = p.is_inf();
    const F ZZ = slots[Par4<F>::sZZ];
    const F Yf = slots[Par4<F>::sY], ZZZf = slots[Par4<F>::sZZZ];
    const F r = F::mul_shared(p.pick(slots[Par4<F>::sX], Yf, Yf, Yf), p.pick(ZZ, ZZZf, ZZZf, ZZZf));
    if (p.lane < 2)
        for (int k = 0; k < F::N; k++) out_jacobian[p.lane * F::N + k] = inf ? 0 : r.l[k];
    if (p.lane == 2)
        for (int k = 0; k < F::N; k++) out_jacobian[2 * F::N + k] = inf ? 0 : ZZ.l[k];
}

// host rows {X, Y, [flag]} at `stride` bytes -> packed {X, Y}; flagged rows become (0,0)
// (reference: Affine_inf_t::mem_t, ec/affine_t.hpp:91-121; stream_t::HtoD pitch copy)
static __global__ void pack_points_kernel(const uint8_t* in, size_t stride, uint32_t words, bool has_flag,
                                   uint32_t* out, uint32_t npoints)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < npoints; i += gridDim.x * blockDim.x) {
        const uint32_t* src = reinterpret_cast<const uint32_t*>(in + (size_t)i * stride);
        bool inf = has_flag && (in[(size_t)i * stride + 4 * words] & 1);
        for (uint32_t k = 0; k < words; k++) out[(size_t)i * words + k] = inf ? 0 : src[k];
    }
}

// ---- precomputed tables (msm_table.cuh) --------------------------------------------------------
template<class F>
__global__ void __launch_bounds__(128)
table_double_kernel(const uint32_t* packed, size_t first, uint32_t n, uint32_t steps, uint32_t copies,
                    uint32_t* xyzz, uint32_t* zzz)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) table_double_body<F>(packed, first, n, steps, copies, xyzz, zzz, i);
}

template<class F>
__global__ void __launch_bounds__(128)
table_normalize_kernel(const uint32_t* xyzz, const uint32_t* zzz_inv, size_t npoints, size_t first, uint32_t n,
                       uint32_t nslots, uint32_t* table)
{
    const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s < nslots) table_normalize_body<F>(xyzz, zzz_inv, npoints, first, n, table, s);
}

// copies 1 .. cfg.copies - 1 of the npoints packed rows at d_table (copy 0) into the rows after them.
// Chunks of at most 2^21 (point, copy) pairs bound the XYZZ scratch (480 MB for 48-byte coordinates).
template<class F>
void build_table(uint32_t* d_table, size_t npoints, const Config& cfg, const stream_t& stream)
{
    const uint32_t K1 = cfg.copies - 1, steps = cfg.wbits * cfg.nwins;
    if (K1 == 0 || npoints == 0) return;
    const size_t chunk = std::min<size_t>(npoints, ((size_t)1 << 21) / K1);
    dev_ptr_t<uint32_t> xyzz(chunk * K1 * 4 * F::N, stream), zzz(chunk * K1 * F::N, stream);
    for (size_t first = 0; first < npoints; first += chunk) {
        const uint32_t n = (uint32_t)std::min(chunk, npoints - first), ns = n * K1;
        table_double_kernel<F><<<(n + 127) / 128, 128, 0, stream>>>(d_table, first, n, steps, cfg.copies, xyzz, zzz);
        pair_invert_kernel<F><<<((ns + PAIR_M - 1) / PAIR_M + 127) / 128, 128, 0, stream>>>(zzz, ns);
        table_normalize_kernel<F><<<(ns + 127) / 128, 128, 0, stream>>>(xyzz, zzz, npoints, first, n, ns, d_table);
        COUNT_LAUNCH(); COUNT_LAUNCH(); COUNT_LAUNCH();
        CUDA_OK(cudaGetLastError());
    }
}

// ---- scalar multiplication of point arrays (msm_scale.cuh) --------------------------------------
template<class F, uint32_t SW>
__global__ void __launch_bounds__(128)
scale_ladder_kernel(const uint32_t* points, const uint32_t* scalars, uint32_t nbits, uint32_t n, uint32_t* xyzz,
                    uint32_t* zzz)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) scale_ladder_body<F, SW>(points, scalars, nbits, xyzz, zzz, i);
}

template<class F>
__global__ void __launch_bounds__(128)
scale_normalize_kernel(const uint32_t* xyzz, const uint32_t* zzz_inv, uint32_t n, uint32_t* out)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) normalize_to_row<F>(xyzz, zzz_inv, i, out + (size_t)i * 2 * F::N);
}

// points per chunk: SCALE_CHUNK, or SPPARK_B200_SCALE_CHUNK (tests: chunk boundaries at small sizes)
inline size_t scale_chunk()
{
    const char* env = getenv("SPPARK_B200_SCALE_CHUNK");
    const size_t v = env ? strtoull(env, nullptr, 10) : 0;
    return v ? std::min(v, SCALE_CHUNK) : SCALE_CHUNK;
}

// d_out[i] = s_i * d_points[i], packed affine rows, enqueued on `stream`; d_out == d_points is allowed
// (a chunk's points are read by its ladder before its normalise writes the same rows)
template<class F>
void scale_points(uint32_t* d_out, const uint32_t* d_points, size_t npoints, const uint32_t* d_scalars,
                  uint32_t scalar_bytes, uint32_t nbits, const stream_t& stream)
{
    if (npoints == 0) return;
    const size_t chunk = std::min(npoints, scale_chunk()), SW = scalar_bytes / 4;
    dev_ptr_t<uint32_t> xyzz(chunk * 4 * F::N, stream), zzz(chunk * F::N, stream);
    for (size_t first = 0; first < npoints; first += chunk) {
        const uint32_t n = (uint32_t)std::min(chunk, npoints - first), blocks = (n + 127) / 128;
        const uint32_t* p = d_points + first * 2 * F::N;
        const uint32_t* s = d_scalars + first * SW;
        switch (SW) {
        case 1: scale_ladder_kernel<F, 1><<<blocks, 128, 0, stream>>>(p, s, nbits, n, xyzz, zzz); break;
        case 2: scale_ladder_kernel<F, 2><<<blocks, 128, 0, stream>>>(p, s, nbits, n, xyzz, zzz); break;
        case 4: scale_ladder_kernel<F, 4><<<blocks, 128, 0, stream>>>(p, s, nbits, n, xyzz, zzz); break;
        default: scale_ladder_kernel<F, 8><<<blocks, 128, 0, stream>>>(p, s, nbits, n, xyzz, zzz); break;
        }
        pair_invert_kernel<F><<<((n + PAIR_M - 1) / PAIR_M + 127) / 128, 128, 0, stream>>>(zzz, n);
        scale_normalize_kernel<F><<<blocks, 128, 0, stream>>>(xyzz, zzz, n, d_out + first * 2 * F::N);
        COUNT_LAUNCH(); COUNT_LAUNCH(); COUNT_LAUNCH();
        CUDA_OK(cudaGetLastError());
    }
}

template<class F>
class msm_t {
    const gpu_t& gpu;
    static constexpr uint32_t PW = 2 * F::N, BW = 4 * F::N, JW = 3 * F::N;   // words per affine/xyzz/jacobian

public:
    explicit msm_t(const gpu_t& g) : gpu(g) {}

    // ---- a transform in flight: buckets persist across slices of points ----------------------
    struct Job {
        Config cfg;                 // window geometry for the WHOLE MSM; npoints = slice capacity
        size_t nslots, slice_cap;
        uint32_t lg_l, items1;
        uint8_t* blob;
        uint32_t *counts, *offsets, *cursor, *ctrl, *heavy_list, *chunk_map, *partials, *sorted, *buckets;
        uint32_t *bin_count, *bin_base, *bin_cur, *overflow;
        uint2* staging;             // the sort's bins: nwins * slice_cap entries of 8 bytes
        uint32_t *R[2], *S[2];
        uint32_t slices_done;
        // batched-affine pre-reduction (msm_pair.cuh), off unless SPPARK_B200_MSM_PAIR=1
        bool pair;
        size_t pair_bound;          // most pair sums one slice can produce
        uint32_t pair_threads;      // threads per forward/backward launch (PAIR_K outputs each)
        uint32_t *counts1, *off1, *wintotal, *winbase, *sums, *pre, *totals;
        // the scratch blob (several GB at 2^26) is released on every exit path, also when a CUDA
        // call between begin() and finish() throws
        cudaStream_t owner;
        Job() : blob(nullptr), owner(nullptr) {}
        Job(const Job&) = delete;
        Job& operator=(const Job&) = delete;
        Job(Job&& o) noexcept { memcpy((void*)this, (const void*)&o, sizeof(Job)); o.blob = nullptr; }
        ~Job() { if (blob) (void)cudaFreeAsync(blob, owner); }
    };

    // total_points and the scalar format fix the window width (make_config); slice_cap is the most
    // points one slice() call may carry
    Job begin(size_t total_points, size_t slice_cap, cudaStream_t stream, uint32_t nbits = 255,
              uint32_t scalar_bytes = 32)
    {
        if (total_points >= (1ull << 31))
            throw cuda_error(-(int)cudaErrorInvalidValue, "msm: npoints must be < 2^31");
        return begin(make_config(total_points, nbits, scalar_bytes), slice_cap, stream);
    }

    // a given geometry (make_config, or config_for_table for the rows of a precomputed table; a batch's
    // group_config of either)
    Job begin(const Config& cfg, size_t slice_cap, cudaStream_t stream)
    {
        Job j;
        CUDA_OK(cudaMallocAsync((void**)&j.blob, plan(j, cfg, slice_cap, nullptr), stream));
        j.owner = stream;
        plan(j, cfg, slice_cap, j.blob);
        g_profile.reset();
        return j;
    }

    // device scratch of a job of geometry cfg over slices of slice_cap points
    static size_t scratch_bytes(const Config& cfg, size_t slice_cap)
    {
        Job j;
        return plan(j, cfg, slice_cap, nullptr);
    }

    // ---- batches: G vectors per job (Config::nvecs), the groups of a batch one after the other -------
    // A group's scratch is G times one vector's (staging, sorted, buckets, running sums: all of it
    // scales with the sets), and its partition keeps G V 2^lg_bins bins open.  G is the largest count
    // that keeps
    //   - the scratch within BATCH_SCRATCH (2 GiB: 5 vectors of 2^20 BLS12-381 G1 points, 39 of 2^16)
    //   - the partition's write frontier G V 2^lg_bins * 128 B within BATCH_FRONTIER (24 MB, under half
    //     of the H100's 50 MB L2, as one vector's 13.6 MB at 2^26 points; 256 KB per vector at 2^20)
    // with the batch then spread evenly over the groups that takes.  G = 1 from BATCH_MAX_POINTS points
    // on: batches were measured faster than a loop of single calls at every shape up to 2^20 points
    // (x1.25 to x20 on an H100 SXM at 700 W, DESIGN.md section 5d), larger ones were not measured.
    // SPPARK_B200_MSM_BATCH_GROUP forces G (tests).
    static constexpr size_t BATCH_SCRATCH = (size_t)2 << 30, BATCH_FRONTIER = (size_t)24 << 20;
    static constexpr size_t BATCH_MAX_POINTS = (size_t)1 << 21;
    static uint32_t group_size(const Config& cfg1, size_t slice_cap, size_t batch)
    {
        if (const char* env = getenv("SPPARK_B200_MSM_BATCH_GROUP"))
            if (atoi(env) > 0) return (uint32_t)std::min<size_t>(batch, (size_t)atoi(env));
        if (batch <= 1 || cfg1.npoints >= BATCH_MAX_POINTS) return 1;
        Config c1 = cfg1;
        c1.npoints = (uint32_t)slice_cap;
        const size_t frontier = ((size_t)c1.nwins << sort_lg_bins(c1, row_stride(c1))) * 128;
        const size_t g = std::min(BATCH_SCRATCH / scratch_bytes(cfg1, slice_cap), BATCH_FRONTIER / frontier);
        // the bucket slots and bins of a group are counted in 32 bits
        const size_t g_slots = ((size_t)1 << 31) / ((size_t)cfg1.nwins << cfg1.lg_nb);
        const size_t gmax = std::max<size_t>(1, std::min({g, g_slots, batch})), ngroups = (batch + gmax - 1) / gmax;
        return (uint32_t)((batch + ngroups - 1) / ngroups);
    }

private:
    // the scratch of a job in one blob: j's geometry and, with a blob, its pointers; returns the bytes
    static size_t plan(Job& j, const Config& cfg, size_t slice_cap, uint8_t* blob)
    {
        j.cfg = cfg;
        j.cfg.npoints = (uint32_t)slice_cap;
        j.slice_cap = slice_cap;
        j.nslots = (size_t)j.cfg.nwins << j.cfg.lg_nb;
        j.lg_l = j.cfg.lg_nb > 12 ? j.cfg.lg_nb - 12 : 0;          // <= 4096 running-sum items per window
        j.items1 = j.cfg.nwins << (j.cfg.lg_nb - j.lg_l);
        j.slices_done = 0;
        const size_t entries = (size_t)j.cfg.nwins * row_stride(j.cfg);
        const size_t heavy_cap = entries / (j.cfg.heavy + 1) + 1;   // most heavy buckets possible
        const size_t chunk_cap = entries / j.cfg.heavy_chunk + heavy_cap; // most chunks possible
        size_t off = 0;
        auto take = [&](size_t bytes) { size_t o = off; off += (bytes + 255) & ~(size_t)255; return o; };
        const size_t o_counts = take(j.nslots * 4), o_offsets = take(j.nslots * 4), o_cursor = take(j.nslots * 4);
        const size_t nbins = (size_t)j.cfg.nwins << sort_lg_bins(j.cfg, row_stride(j.cfg));
        const size_t o_bcount = take(nbins * 4), o_bbase = take(nbins * 4), o_bcur = take(nbins * 4), o_over = take(nbins * 4);
        const size_t o_staging = take(entries * 8);
        const size_t o_ctrl = take(16), o_heavy = take(heavy_cap * 12), o_cmap = take(chunk_cap * 4);
        const size_t o_partials = take(chunk_cap * BW * 4);
        const size_t o_sorted = take(entries * 4);
        const size_t o_buckets = take(j.nslots * BW * 4);
        const size_t o_r0 = take((size_t)j.items1 * BW * 4), o_s0 = take((size_t)j.items1 * BW * 4);
        const size_t o_r1 = take((size_t)j.items1 * BW * 4 / 2 + 4096), o_s1 = take((size_t)j.items1 * BW * 4 / 2 + 4096);
        // experimental, measured once in round 1 (DESIGN.md section 8): halves the bucket lists with
        // batched affine pair sums before the XYZZ accumulation
        const char* pair_env = getenv("SPPARK_B200_MSM_PAIR");
        j.pair = pair_env && atoi(pair_env) != 0 && entries + j.nslots < (1ull << 31);
        j.pair_bound = (entries + std::min<size_t>(entries, j.nslots) + 1) / 2;
        j.pair_threads = (uint32_t)std::min<size_t>((j.pair_bound + PAIR_K - 1) / PAIR_K, (size_t)1 << 21);
        size_t o_c1 = 0, o_o1 = 0, o_wt = 0, o_wb = 0, o_sums = 0, o_pre = 0, o_tot = 0;
        if (j.pair) {
            o_c1 = take(j.nslots * 4); o_o1 = take(j.nslots * 4);
            o_wt = take((j.cfg.nwins + 1) * 4); o_wb = take((j.cfg.nwins + 1) * 4);
            o_sums = take(j.pair_bound * 2 * F::N * 4);
            o_pre = take((size_t)j.pair_threads * PAIR_K * F::N * 4);
            o_tot = take((size_t)j.pair_threads * F::N * 4);
        }
        if (!blob) return off;
        auto U32 = [&](size_t o) { return reinterpret_cast<uint32_t*>(blob + o); };
        j.counts = U32(o_counts); j.offsets = U32(o_offsets); j.cursor = U32(o_cursor);
        j.ctrl = U32(o_ctrl); j.heavy_list = U32(o_heavy); j.chunk_map = U32(o_cmap);
        j.partials = U32(o_partials); j.sorted = U32(o_sorted); j.buckets = U32(o_buckets);
        j.bin_count = U32(o_bcount); j.bin_base = U32(o_bbase); j.bin_cur = U32(o_bcur); j.overflow = U32(o_over);
        j.staging = reinterpret_cast<uint2*>(blob + o_staging);
        j.R[0] = U32(o_r0); j.S[0] = U32(o_s0); j.R[1] = U32(o_r1); j.S[1] = U32(o_s1);
        j.counts1 = U32(o_c1); j.off1 = U32(o_o1); j.wintotal = U32(o_wt); j.winbase = U32(o_wb);
        j.sums = U32(o_sums); j.pre = U32(o_pre); j.totals = U32(o_tot);
        return off;
    }

public:
    // fold `n` (<= slice_cap) device-resident points/scalars into the buckets
    void slice(Job& j, const uint32_t* d_points, const uint32_t* d_scalars, size_t n, cudaStream_t stream)
    {
        if (n == 0) return;
        Config cfg = j.cfg;
        cfg.npoints = (uint32_t)n;
        cfg.merge = j.slices_done ? 1 : 0;
        const uint32_t sms = (uint32_t)gpu.sm_count();
        g_profile.mark("sort", stream);
        const SortBufs sb{j.counts, j.offsets, j.cursor, j.ctrl, j.heavy_list, j.chunk_map, j.sorted,
                          j.bin_count, j.bin_base, j.bin_cur, j.overflow, j.staging};
        sort_slice(cfg, SORT_CAP, d_scalars, sb, sms, stream);

        g_profile.mark("accumulate", stream);
        int occ = 1;
        CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, accumulate_kernel<F>, ACC_THREADS, 0));
        if (occ < 1) occ = 1;
        size_t want = (j.nslots + ACC_THREADS - 1) / ACC_THREADS;
        uint32_t acc_blocks = (uint32_t)std::min<size_t>(want, (size_t)sms * occ);
        if (j.pair) {
            const uint32_t nslots = (uint32_t)j.nslots;
            pair_counts_kernel<<<sms * 8, 256, 0, stream>>>(cfg, j.counts, j.counts1, nslots);
            pair_scan_kernel<<<cfg.nwins, 1024, 0, stream>>>(cfg, j.counts1, j.off1, j.wintotal);
            pair_winbase_kernel<<<1, 32, 0, stream>>>(cfg, j.wintotal, j.winbase);
            // the host does not know how many pair sums this slice has (winbase[nwins], on the
            // device): launches cover the bound, threads past the real total return at once
            const size_t ent = (size_t)cfg.nwins * row_stride(cfg);
            const size_t bound = (ent + std::min<size_t>(ent, j.nslots) + 1) / 2;
            const size_t per_launch = (size_t)j.pair_threads * PAIR_K;
            for (size_t o0 = 0; o0 < bound; o0 += per_launch) {
                const uint32_t nth = (uint32_t)std::min<size_t>(j.pair_threads, (bound - o0 + PAIR_K - 1) / PAIR_K);
                pair_forward_kernel<F><<<(nth + 127) / 128, 128, 0, stream>>>(
                    cfg, d_points, j.sorted, j.offsets, j.counts, j.counts1, j.off1, j.winbase, (uint32_t)o0, nth, j.pre, j.totals);
                pair_invert_kernel<F><<<((nth + PAIR_M - 1) / PAIR_M + 127) / 128, 128, 0, stream>>>(j.totals, nth);
                pair_backward_kernel<F><<<(nth + 127) / 128, 128, 0, stream>>>(
                    cfg, d_points, j.sorted, j.offsets, j.counts, j.counts1, j.off1, j.winbase, (uint32_t)o0, nth, j.pre, j.totals, j.sums);
                COUNT_LAUNCH(); COUNT_LAUNCH(); COUNT_LAUNCH();
            }
            CUDA_OK(cudaGetLastError());
            g_profile.mark("accumulate_sums", stream);
            accumulate_direct_kernel<F><<<acc_blocks, ACC_THREADS, 0, stream>>>(cfg, j.sums, j.offsets, j.counts, j.buckets,
                                                                               j.ctrl, j.counts1, j.off1, j.winbase);
        } else {
            accumulate_kernel<F><<<acc_blocks, ACC_THREADS, 0, stream>>>(cfg, d_points, j.sorted, j.offsets, j.counts,
                                                                        j.buckets, j.ctrl);
        }
        COUNT_LAUNCH();
        g_profile.mark("heavy", stream);
        heavy_chunks_kernel<F><<<sms * 4, HEAVY_THREADS, HEAVY_THREADS * BW * 4, stream>>>(
            cfg, d_points, j.sorted, j.offsets, j.counts, j.ctrl, j.heavy_list, j.chunk_map, j.partials);
        COUNT_LAUNCH();
        heavy_fold_kernel<F><<<sms, HEAVY_THREADS, HEAVY_THREADS * BW * 4, stream>>>(cfg, j.ctrl, j.heavy_list,
                                                                                    j.partials, j.buckets);
        COUNT_LAUNCH();
        CUDA_OK(cudaGetLastError());
        if (getenv("SPPARK_B200_MSM_DEBUG")) {
            uint32_t dbg[3];
            CUDA_OK(cudaMemcpyAsync(dbg, j.ctrl, 12, cudaMemcpyDeviceToHost, stream));
            CUDA_OK(cudaStreamSynchronize(stream));
            fprintf(stderr, "[msm] slice %u n=%u wbits=%u nwins=%u heavy_thr=%u tasks_claimed=%u nheavy=%u nchunks=%u acc_blocks=%u"
                    " digits=%u sets=%u copies=%u nbits=%u sbytes=%u vecs=%u vsets=%u\n",
                    j.slices_done, cfg.npoints, cfg.wbits, cfg.nwins, cfg.heavy, dbg[0], dbg[1], dbg[2], acc_blocks,
                    digit_count(cfg), cfg.nwins, cfg.copies, (uint32_t)cfg.nbits, 4u * cfg.swords, cfg.nvecs, vec_sets(cfg));
        }
        j.slices_done++;
    }

    // running sums over the buckets, Horner over the windows -> d_out (JW words per vector), frees the job
    void finish(Job& j, uint32_t* d_out, cudaStream_t stream)
    {
        if (j.slices_done == 0) {
            CUDA_OK(cudaMemsetAsync(d_out, 0, (size_t)j.cfg.nvecs * JW * 4, stream));
        } else {
            const Config& cfg = j.cfg;
            g_profile.mark("reduce", stream);
            reduce1_kernel<F><<<(j.items1 + 127) / 128, 128, 0, stream>>>(cfg, j.buckets, j.lg_l, j.items1, j.R[0], j.S[0]);
            COUNT_LAUNCH();
            uint32_t per_win = 1u << (cfg.lg_nb - j.lg_l), lg_span = j.lg_l, cur = 0;
            while (per_win > 1) {
                uint32_t lg_g = 31 - __builtin_clz(per_win);
                if (lg_g > 4) lg_g = 4;                         // radix 16 keeps the serial chains short
                uint32_t G = 1u << lg_g, nitems = cfg.nwins * (per_win >> lg_g);
                constexpr uint32_t PG = par_groups<F>::value;
                combine_par_kernel<F><<<(nitems + PG - 1) / PG, 4 * PG, 0, stream>>>(j.R[cur], j.S[cur], G, lg_span, nitems,
                                                                                     j.R[cur ^ 1], j.S[cur ^ 1]);
                COUNT_LAUNCH();
                per_win >>= lg_g;
                lg_span += lg_g;
                cur ^= 1;
            }
            g_profile.mark("finish", stream);
            finish_par_kernel<F><<<cfg.nvecs, 32, 0, stream>>>(cfg, j.R[cur], d_out);
            COUNT_LAUNCH();
            g_profile.mark("end", stream);
            CUDA_OK(cudaGetLastError());
        }
        CUDA_OK(cudaFreeAsync(j.blob, stream));
        j.blob = nullptr;
    }

    // all inputs device-resident: d_points packed affine, d_scalars `batch` vectors of npoints scalars of
    // scalar_bytes each (bits from nbits up ignored), run in groups of group_size vectors.  d_out: batch
    // * JW words of device memory.  Enqueues on `stream`; no synchronisation.
    void invoke_dev(uint32_t* d_out, const uint32_t* d_points, size_t npoints,
                    const uint32_t* d_scalars, cudaStream_t stream, uint32_t nbits = 255, uint32_t scalar_bytes = 32,
                    size_t batch = 1)
    {
        if (npoints == 0) {
            CUDA_OK(cudaMemsetAsync(d_out, 0, batch * JW * 4, stream));
            return;
        }
        if (npoints >= (1ull << 31))
            throw cuda_error(-(int)cudaErrorInvalidValue, "msm: npoints must be < 2^31");
        const Config cfg1 = make_config(npoints, nbits, scalar_bytes);
        const size_t G = group_size(cfg1, npoints, batch), sw = scalar_bytes / 4;
        for (size_t b0 = 0; b0 < batch; b0 += G) {
            const uint32_t g = (uint32_t)std::min(G, batch - b0);
            Job j = begin(group_config(cfg1, g), npoints, stream);
            slice(j, d_points, d_scalars + b0 * npoints * sw, npoints, stream);
            finish(j, d_out + b0 * JW, stream);
        }
    }
};

}  // namespace msm
