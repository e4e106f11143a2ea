// class NTT<F>: the reference's `class NTT` (ntt/ntt.cuh:31-366) for single-word fields,
// rebuilt on the pass kernel of ntt_core.cuh.  Same public entry points and semantics:
//   NTT::Base(gpu, host_inout, lg, order, direction, type)        ntt/ntt.cuh:216-244
//   NTT::Base_dev_ptr(stream, d_inout, lg, order, direction, type) ntt/ntt.cuh:344-350
// order/direction/type are the reference enums (ntt/ntt.cuh:33-35).
#pragma once
#include "../util/gpu.cuh"
#include "ntt_plan.hpp"
#include "ntt_warp.cuh"

namespace ntt {

template<class F>
__global__ void __launch_bounds__(F::NTT_MAX_THREADS)
pass_kernel(const Pass d, const Tables<F> tb, const typename F::T* in, typename F::T* out)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    typename F::T* smem = reinterpret_cast<typename F::T*>(smem_raw);
    const uint32_t tid = threadIdx.x, nthreads = blockDim.x, t = blockIdx.x;
    const KDyn k{d};

    phase_twiddles<F>(k, tb, smem, tid, nthreads);
    phase_load<F>(k, d, tb, in, smem, t, tid, nthreads);
    __syncthreads();
    const uint32_t nsteps = step_count<F>(d.lg_r);
    for (uint32_t s = 0; s < nsteps; s++) {
        phase_step_dyn<F>(k, smem, s * F::LG_EPT, step_log_e<F>(d.lg_r, s), tid);
        __syncthreads();
    }
    phase_store<F>(k, d, tb, out, smem, t, tid, nthreads);
}

// the same pass with its shape fixed at compile time (see KStat in ntt_core.cuh)
template<class F, class K>
__global__ void __launch_bounds__(F::NTT_MAX_THREADS)
pass_kernel_static(const Pass d, const Tables<F> tb, const typename F::T* in, typename F::T* out, uint32_t ntiles)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    typename F::T* smem = reinterpret_cast<typename F::T*>(smem_raw);
    const uint32_t tid = threadIdx.x;
    constexpr uint32_t R = K::lg_r();
    constexpr uint32_t LG_EPT = F::LG_EPT;
    constexpr uint32_t nthreads = (R >= LG_EPT ? (1u << (R - LG_EPT)) : 1u) << K::lg_w();
    const K k(d);

    // persistent CTAs: the sub-NTT twiddles (2^R words, a quarter of a tile's bytes) are staged into
    // shared memory once per CTA, by ONE bulk asynchronous copy (TMA, cp.async.bulk) that runs
    // while the first tile is being loaded; every thread waits on the copy's mbarrier before the
    // first butterfly step
    __shared__ uint64_t tw_bar;
    typename F::T* tw_dst = smem + (col_stride(R) << K::lg_w());
    if (tid == 0) mbar_init(&tw_bar, 1);
    __syncthreads();
    if (tid == 0) tma_load_1d(tw_dst, tb.dense, (uint32_t)(sizeof(typename F::T) << R), &tw_bar);
    bool tw_pending = true;
    for (uint32_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
        phase_load<F>(k, d, tb, in, smem, t, tid, nthreads);
        if (tw_pending) { mbar_wait(&tw_bar, 0); tw_pending = false; }
        __syncthreads();
#pragma unroll
        for (uint32_t s = 0; s < step_count<F>(R); s++) {
            constexpr uint32_t full = R / LG_EPT;
            if (s < full) phase_step<F, K, LG_EPT>(k, smem, s * LG_EPT, tid);
            else phase_step_dyn<F>(k, smem, s * LG_EPT, R - full * LG_EPT, tid);
            __syncthreads();
        }
        phase_store<F>(k, d, tb, out, smem, t, tid, nthreads);
        __syncthreads();
    }
}

// a pass over the columns of a row-major matrix (set_matrix, phase_load_matrix in ntt_core.cuh):
// persistent CTAs walk the tiles i = t * ncb + cb (transform tile t, column block cb), so that
// neighbouring CTAs read neighbouring column blocks of the same rows.  The sub-NTT twiddles are
// staged once per CTA, by one bulk asynchronous copy (TMA) under the first tile load when the table
// is whole 16-byte units, by the threads otherwise (sub-NTTs of 2 or 4 BabyBear words).  K is KDyn
// (any shape) or KShape<R, W>.
template<class F, class K>
__global__ void __launch_bounds__(F::NTT_MAX_THREADS)
matrix_pass_kernel(const Pass d, const Tables<F> tb, const typename F::T* in, typename F::T* out,
                   uint64_t width, uint64_t ncb, uint64_t ntiles)
{
    typedef typename F::T T;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    T* smem = reinterpret_cast<T*>(smem_raw);
    const uint32_t tid = threadIdx.x;
    constexpr uint32_t LG_EPT = F::LG_EPT;
    const K k{d};
    const uint32_t R = k.lg_r();
    const uint32_t nthreads = (R >= LG_EPT ? (1u << (R - LG_EPT)) : 1u) << k.lg_w();

    __shared__ uint64_t tw_bar;
    const uint32_t tw_bytes = (uint32_t)sizeof(T) << R;
    const bool tma = tw_bytes % 16 == 0;
    if (tma) {
        if (tid == 0) mbar_init(&tw_bar, 1);
        __syncthreads();
        if (tid == 0) tma_load_1d(smem + (col_stride(R) << k.lg_w()), tb.dense, tw_bytes, &tw_bar);
    } else {
        phase_twiddles<F>(k, tb, smem, tid, nthreads);
    }
    bool tw_pending = tma;
    for (uint64_t i = blockIdx.x; i < ntiles; i += gridDim.x) {
        const uint64_t t = i / ncb, cb = i - t * ncb;
        phase_load_matrix<F>(k, d, tb, in, smem, t, cb, width, tid, nthreads);
        if (tw_pending) { mbar_wait(&tw_bar, 0); tw_pending = false; }
        __syncthreads();
#pragma unroll
        for (uint32_t s = 0; s < step_count<F>(R); s++) {
            if (s < R / LG_EPT) phase_step<F, K, LG_EPT>(k, smem, s * LG_EPT, tid);
            else phase_step_dyn<F>(k, smem, s * LG_EPT, R - (R / LG_EPT) * LG_EPT, tid);
            __syncthreads();
        }
        phase_store_matrix<F>(k, d, tb, out, smem, t, cb, width, tid, nthreads);
        __syncthreads();
    }
}

// one launch of matrix_pass_kernel<F, K>: as many CTAs as fit on the GPU at once, at most one per tile
template<class F, class K>
void launch_matrix_pass(const Pass& d, const Tables<F>& tb, const typename F::T* in, typename F::T* out,
                        uint64_t width, uint32_t lg_n, cudaStream_t stream)
{
    int dev = 0;
    CUDA_OK(cudaGetDevice(&dev));
    smem_opt_in<matrix_pass_kernel<F, K>>(dev, 226 * 1024);      // + the static mbarrier word <= 227 KiB
    static int sms_of[64];
    if (!sms_of[dev & 63]) CUDA_OK(cudaDeviceGetAttribute(&sms_of[dev & 63], cudaDevAttrMultiProcessorCount, dev));
    const size_t smem = smem_elems(d) * sizeof(typename F::T);
    const uint32_t threads = tile_threads<F>(d);
    const uint64_t ncb = matrix_col_blocks(d, width), ntiles = ncb << (lg_n - d.lg_r);
    uint32_t per_sm = smem <= 48 * 1024 ? 4 : smem <= 100 * 1024 ? 2 : 1;
    while (per_sm > 1 && per_sm * threads > 2048) per_sm >>= 1;
    const uint64_t cap = (uint64_t)sms_of[dev & 63] * per_sm;
    matrix_pass_kernel<F, K><<<(uint32_t)(ntiles < cap ? ntiles : cap), threads, smem, stream>>>(
        d, tb, in, out, width, ncb, ntiles);
}

// launcher table for the statically shaped passes; returns false if (d) has no static twin
template<class F> bool launch_static(const Pass& d, const Tables<F>& tb, const typename F::T* in,
                                     typename F::T* out, uint32_t ntiles, size_t smem, cudaStream_t stream);
// a matrix pass: the statically shaped kernel of d's (lg_r, lg_w) if there is one, else the
// run-time shaped one (ntt.cu)
template<class F> void launch_matrix(const Pass& d, const Tables<F>& tb, const typename F::T* in, typename F::T* out,
                                     uint64_t width, uint32_t lg_n, cudaStream_t stream);
// warp-autonomous pass (ntt_warp.cuh) for 4 <= d.lg_r <= 8, single-word fields; false otherwise
template<class F> bool launch_warp(const gpu_t& gpu, const Pass& d, const Tables<F>& tb, const typename F::T* in,
                                   typename F::T* out, uint32_t ncols, cudaStream_t stream);

// ---- one-time table generation (role of NTTParameters, ntt/parameters.cuh:147-337) ----
template<class F>
__global__ void gen_tables_kernel(typename F::T* dense, typename F::T* tlo, typename F::T* thi,
                                  uint32_t n_hi, uint32_t lg_n, bool inverse)
{
    typedef typename F::T T;
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    T w_max = F::root_of_unity_max();
    if (inverse) w_max = F::inv(w_max);
    // w_(2^lg) = w_max^(2^(MAX_LG - lg))
    if (i < (1u << LG_DENSE)) {
        if (i == 0) {
            dense[0] = F::one();
        } else {
            uint32_t lg_h = 31 - __clz(i), idx = i - (1u << lg_h);     // i = h + idx
            T w = F::pow(w_max, 1ull << (F::MAX_LG - (lg_h + 1)));
            dense[i] = F::pow(w, idx);
        }
    }
    T wn = F::pow(w_max, 1ull << (F::MAX_LG - lg_n));
    if (i < (1u << LG_TLO)) tlo[i] = F::pow(wn, i);
    if (i < n_hi) thi[i] = F::pow(wn, (uint64_t)i << LG_TLO);
}

// twist tables of the warp-autonomous passes (ntt_warp.cuh): for R = 5..8,
// mid[mid_offset(R) + k0 * L + b] = w_(2^R)^(b * k0), L = 2^(R-4), k0 < 16, b < L
template<class F>
__global__ void gen_mid_kernel(typename F::T* mid, bool inverse)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= MID_WORDS) return;
    uint32_t R = 5;
    while (R < WARP_MAX_LG_R && i >= mid_offset(R + 1)) R++;
    if ((uint32_t)F::MAX_LG < R) { mid[i] = F::one(); return; }
    const uint32_t L = 1u << (R - 4), e = i - mid_offset(R), k0 = e / L, b = e % L;
    typename F::T w_max = F::root_of_unity_max();
    if (inverse) w_max = F::inv(w_max);
    mid[i] = F::pow(F::pow(w_max, 1ull << (F::MAX_LG - R)), (uint64_t)b * k0);
}

// coset: x[i] *= g^nat(i)   (reference: LDE_distribute_powers, ntt/kernels.cu:131-153)
template<class F>
__global__ void gen_coset_kernel(typename F::T* g0, typename F::T* g1, typename F::T* g2, bool inverse)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    typename F::T g = F::group_gen();
    if (inverse) g = F::inv(g);
    if (i < 4096) { g0[i] = F::pow(g, i); g1[i] = F::pow(g, (uint64_t)i << 12); }
    if (i < 256) g2[i] = F::pow(g, (uint64_t)i << 24);
}

// over a batch of transforms of 2^lg_n elements each: `count` = batch << lg_n elements, the
// exponent is taken within each transform
template<class F>
__global__ void coset_kernel(typename F::T* data, uint32_t lg_n, bool bitrev,
                             const typename F::T* g0, const typename F::T* g1,
                             const typename F::T* g2, size_t count)
{
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < count;
         i += (size_t)gridDim.x * blockDim.x)
        data[i] = F::canon(coset_mul<F>(F::load(data[i]), i, lg_n, bitrev, g0, g1, g2));
}

// LDE: zero-stuffing blow-up fused with the coset shift (reference:
// LDE_spread_distribute_powers, ntt/kernels.cu:155-237).  `in` holds the n coefficients in
// bit-reversed order (the output of an NR inverse transform); out[i << lg_blowup] = in[i] *
// g^bitrev(i), every other slot of the (n << lg_blowup)-element array is zero -- i.e. the
// coefficients of P(g*x) in the bit-reversed order of the extended domain.
// out[brev(i)] = in[i]: the natural-order copy of a bit-reversed array (LDE_aux's coefficients)
template<class F>
__global__ void bitrev_copy_kernel(typename F::T* out, const typename F::T* in, uint32_t lg_n)
{
    const size_t n = (size_t)1 << lg_n;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        out[brev32((uint32_t)i, lg_n)] = in[i];
}

template<class F>
__global__ void lde_spread_kernel(typename F::T* out, const typename F::T* in, uint32_t lg_n, uint32_t lg_blowup,
                                  const typename F::T* g0, const typename F::T* g1, const typename F::T* g2,
                                  bool shift = true, size_t batch = 1)
{
    // a batch: `batch` rows of 2^lg_n in, rows of 2^(lg_n + lg_blowup) out; row r's slot i << lg_blowup
    // is element (r << (lg_n + lg_blowup)) + (i << lg_blowup) = (global input index) << lg_blowup
    typedef typename F::T T;
    const size_t n_ext = batch << (lg_n + lg_blowup);
    const uint32_t mask = (1u << lg_blowup) - 1;
    T zero = F::sub(F::one(), F::one());
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n_ext; i += (size_t)gridDim.x * blockDim.x) {
        T x = zero;
        if ((i & mask) == 0) {
            const size_t src = i >> lg_blowup;
            x = F::load(in[src]);
            if (shift) x = coset_mul<F>(x, src, lg_n, true, g0, g1, g2);
            x = F::canon(x);
        }
        out[i] = x;
    }
}

// coset shift and LDE spread of a row-major matrix (coset_matrix_row, lde_spread_matrix_row): a block
// of bx x by threads, bx (a power of two) along a row's columns, by rows at a time; one coset factor
// per row and thread, no division per element
template<class F>
__global__ void coset_matrix_kernel(typename F::T* data, uint32_t lg_n, uint64_t width, bool bitrev,
                                    const typename F::T* g0, const typename F::T* g1, const typename F::T* g2)
{
    const uint64_t rows = (uint64_t)1 << lg_n;
    for (uint64_t r = (uint64_t)blockIdx.x * blockDim.y + threadIdx.y; r < rows; r += (uint64_t)gridDim.x * blockDim.y)
        coset_matrix_row<F>(data, r, width, lg_n, bitrev, g0, g1, g2, threadIdx.x, blockDim.x);
}

template<class F>
__global__ void lde_spread_matrix_kernel(typename F::T* out, const typename F::T* in, uint32_t lg_n, uint32_t lg_blowup,
                                         uint64_t width, const typename F::T* g0, const typename F::T* g1,
                                         const typename F::T* g2)
{
    const uint64_t rows = (uint64_t)1 << (lg_n + lg_blowup);
    for (uint64_t r = (uint64_t)blockIdx.x * blockDim.y + threadIdx.y; r < rows; r += (uint64_t)gridDim.x * blockDim.y)
        lde_spread_matrix_row<F>(out, in, r, width, lg_n, lg_blowup, g0, g1, g2, threadIdx.x, blockDim.x);
}

template<class F> struct FieldId;     // specialised in ntt.cu: cache key + shared-memory tile
template<class F> struct NTTMatrix;

template<class F>
class NTT {
    typedef typename F::T T;
    friend struct NTTMatrix<F>;       // shares the twiddle and coset tables
public:
    enum class InputOutputOrder { NN, NR, RN, RR, BB };
    enum class Direction { forward, inverse };
    enum class Type { standard, coset };

private:
    struct DevTables { Tables<F> view; };

    static uint64_t key(uint32_t kind, uint32_t lg_n, bool inverse)
    {   return ((uint64_t)FieldId<F>::id << 48) | ((uint64_t)kind << 40) | ((uint64_t)lg_n << 8) | inverse;   }

    // twiddles live for the life of the process, per device (as NTTParameters::all does)
    static const Tables<F>& tables(const gpu_t& gpu, uint32_t lg_n, bool inverse, cudaStream_t stream)
    {
        std::lock_guard<std::mutex> lock(const_cast<gpu_t&>(gpu).cache_mtx);
        auto& cache = const_cast<gpu_t&>(gpu).cache;
        auto it = cache.find(key(0, lg_n, inverse));
        if (it != cache.end()) return *reinterpret_cast<Tables<F>*>(it->second);

        const uint32_t n_hi = lg_n > LG_TLO ? 1u << (lg_n - LG_TLO) : 1;
        const size_t total = (1u << LG_DENSE) + (1u << LG_TLO) + 512 + n_hi;
        T* blob;
        CUDA_OK(cudaMalloc(&blob, total * sizeof(T)));
        // mid sits before thi: its sub-tables are sources of 16-byte aligned bulk copies
        T *dense = blob, *tlo = blob + (1u << LG_DENSE), *mid = tlo + (1u << LG_TLO), *thi = mid + 512;
        uint32_t nthr = n_hi > 4096 ? n_hi : 4096;
        gen_tables_kernel<F><<<(nthr + 255) / 256, 256, 0, stream>>>(dense, tlo, thi, n_hi, lg_n, inverse);
        COUNT_LAUNCH();
        gen_mid_kernel<F><<<(MID_WORDS + 255) / 256, 256, 0, stream>>>(mid, inverse);
        COUNT_LAUNCH();
        CUDA_OK(cudaGetLastError());
        CUDA_OK(cudaStreamSynchronize(stream));      // one-time: other streams may use it next
        T half = F::inv(F::add(F::one(), F::one())), ninv = F::one();
        for (uint32_t i = 0; i < lg_n; i++) ninv = F::mul(ninv, half);
        auto* tb = new Tables<F>{dense, tlo, thi, ninv, mid, {}};
        if ((uint32_t)F::MAX_LG >= 4) {
            T w_max = F::root_of_unity_max();
            if (inverse) w_max = F::inv(w_max);
            const T w16 = F::pow(w_max, 1ull << (F::MAX_LG - 4));
            tb->w16[0] = F::one();
            for (uint32_t i = 1; i < 8; i++) tb->w16[i] = F::mul(tb->w16[i - 1], w16);
        }
        cache[key(0, lg_n, inverse)] = tb;
        return *tb;
    }

    struct CosetTables { T *g0, *g1, *g2; };
    static const CosetTables& coset_tables(const gpu_t& gpu, bool inverse, cudaStream_t stream)
    {
        std::lock_guard<std::mutex> lock(const_cast<gpu_t&>(gpu).cache_mtx);
        auto& cache = const_cast<gpu_t&>(gpu).cache;
        auto it = cache.find(key(1, 0, inverse));
        if (it != cache.end()) return *reinterpret_cast<CosetTables*>(it->second);
        T* blob;
        CUDA_OK(cudaMalloc(&blob, (4096 + 4096 + 256) * sizeof(T)));
        auto* ct = new CosetTables{blob, blob + 4096, blob + 8192};
        gen_coset_kernel<F><<<16, 256, 0, stream>>>(ct->g0, ct->g1, ct->g2, inverse);
        COUNT_LAUNCH();
        CUDA_OK(cudaGetLastError());
        CUDA_OK(cudaStreamSynchronize(stream));
        cache[key(1, 0, inverse)] = ct;
        return *ct;
    }

    static void coset_scale(const gpu_t& gpu, T* d_inout, uint32_t lg_n, bool bitrev, bool inverse,
                            cudaStream_t stream, size_t batch = 1)
    {
        const CosetTables& ct = coset_tables(gpu, inverse, stream);
        size_t n = batch << lg_n;
        size_t blocks = (n + 255) / 256;
        size_t cap = (size_t)gpu.sm_count() * 16;
        coset_kernel<F><<<(uint32_t)(blocks < cap ? blocks : cap), 256, 0, stream>>>(d_inout, lg_n, bitrev, ct.g0, ct.g1, ct.g2, n);
        COUNT_LAUNCH();
        CUDA_OK(cudaGetLastError());
    }

    // Which pass kernel: below 2^20 elements the warp-autonomous passes (ntt_warp.cuh: no block
    // barrier, any number of warps busy) win; from 2^20 on the two 12-stage block-tile passes move
    // a third less data (the crossover was chosen on an earlier GPU and has not been re-measured
    // on H100).  SPPARK_B200_NTT_WARP=1 /
    // SPPARK_B200_NTT_BLOCK=1 force one or the other (experiments, tests).
    static bool use_warp_path(uint32_t lg_n)
    {
        if (F::LG_EPT != 4 || lg_n < WARP_MIN_LG_R) return false;
        const char* b = getenv("SPPARK_B200_NTT_BLOCK");
        const char* w = getenv("SPPARK_B200_NTT_WARP");
        if (b && b[0] == '1') return false;
        if (w && w[0] == '1') return true;
        return lg_n < 20;
    }

public:
    // device-resident transform, enqueued on `stream`, no synchronisation.  batch > 1: `batch`
    // transforms of 2^lg_n elements stored one after another, one plan and one launch per pass for
    // all of them
    static void NTT_internal(const gpu_t& gpu, T* d_inout, uint32_t lg_n, InputOutputOrder order,
                             Direction direction, Type type, cudaStream_t stream, size_t batch = 1)
    {
        if (lg_n == 0 || batch == 0) return;
        if (lg_n > (uint32_t)F::MAX_LG || lg_n > 30)
            throw cuda_error(-(int)cudaErrorInvalidValue, "NTT: lg_domain_size out of range");
        const bool inverse = direction == Direction::inverse;
        // coset exponents follow the reference's `bitrev` flags exactly (ntt/ntt.cuh:174-209):
        // for RR they are bit-reversed although the data is in natural order.
        const bool in_rev = order != InputOutputOrder::NN && order != InputOutputOrder::NR;
        const bool out_rev = order != InputOutputOrder::NN && order != InputOutputOrder::RN;

        // single-word fields: warp-autonomous passes of 2^4..2^8-point sub-NTTs (ntt_warp.cuh);
        // 256-bit fields (and SPPARK_B200_NTT_BLOCK=1): block-tile passes of up to 2^12 points.  A
        // warp-path tile holds up to 64 adjacent columns; the block tiles are sized from all the
        // transforms of a batch together
        const bool warp_path = use_warp_path(lg_n);
        const uint32_t lg_tile = warp_path ? WARP_MAX_LG_R + 6
                                           : block_lg_tile(lg_n, batch, FieldId<F>::lg_tile, getenv("SPPARK_B200_NTT_LG_TILE"));
        Plan plan = make_plan(lg_n, (int)order, inverse, lg_tile, 6, warp_path ? WARP_MAX_LG_R : F::NTT_MAX_LG_R);
        if (batch > 1) {
            if (!set_batch(plan, batch))
                throw cuda_error(-(int)cudaErrorInvalidValue, "NTT: this plan cannot be batched");
            // the tiles of the whole batch index one grid (the warp passes go in launches of < 2^31
            // elements, below)
            for (const Pass& d : plan.passes)
                if ((batch << (lg_n - d.lg_r - d.lg_w)) > 0x7fffffffull)
                    throw cuda_error(-(int)cudaErrorInvalidValue, "NTT: batch too large for this lg_domain_size");
        }

        if (!inverse && type == Type::coset)
            coset_scale(gpu, d_inout, lg_n, in_rev, false, stream, batch);

        const Tables<F>& tb = tables(gpu, lg_n, inverse, stream);

        T* scratch = nullptr;
        if (plan.needs_scratch)
            CUDA_OK(cudaMallocAsync((void**)&scratch, (sizeof(T) * batch) << lg_n, stream));
        T* buf[2] = {d_inout, scratch};

        smem_opt_in<pass_kernel<F>>(gpu.cid(), (int)gpu.props().sharedMemPerBlockOptin);
        g_profile.reset();
        for (const Pass& d : plan.passes) {
            g_profile.mark("pass", stream);
            uint32_t ntiles = (uint32_t)(batch << (lg_n - d.lg_r - d.lg_w));
            size_t smem = smem_elems(d) * sizeof(T);
            bool done = false;
            if constexpr (F::LG_EPT == 4) {
                if (warp_path) {
                    // the warp passes address a launch's elements in 32 bits: a batch past 2^31
                    // elements goes in launches of whole rows, each on its own slice of the buffers
                    const size_t rows = std::max<size_t>(1, ((size_t)1 << 31) >> lg_n);
                    done = true;
                    for (size_t r0 = 0; r0 < batch && done; r0 += rows) {
                        const size_t off = r0 << lg_n, nr = std::min(rows, batch - r0);
                        done = launch_warp<F>(gpu, d, tb, buf[d.src] + off, buf[d.dst] + off,
                                              (uint32_t)(nr << (lg_n - d.lg_r)), stream);
                    }
                }
            }
            if (!done && !launch_static<F>(d, tb, buf[d.src], buf[d.dst], ntiles, smem, stream))
                pass_kernel<F><<<ntiles, tile_threads<F>(d), smem, stream>>>(d, tb, buf[d.src], buf[d.dst]);
            COUNT_LAUNCH();
            CUDA_OK(cudaGetLastError());
        }
        g_profile.mark("end", stream);
        if (scratch) CUDA_OK(cudaFreeAsync(scratch, stream));

        if (inverse && type == Type::coset)
            coset_scale(gpu, d_inout, lg_n, out_rev, true, stream, batch);
    }

    // one local stage of the slab-sharded transform (ntt_plan.hpp: make_slab_plan); which = 1:
    // d_in [N1][N2/G] -> d_out = all-to-all staging [G][N2/G][N1/G]; which = 2: d_in = the received
    // [N2][N1/G] matrix, transformed down its columns with the result left in d_in; d_out is
    // scratch of the same size, touched only when N2 needs more than one pass (it may equal d_in
    // otherwise).  Enqueued on `stream`.
    // peers != nullptr (which = 1 only): fused exchange -- 2^lg_g device pointers, peers[q] = rank
    // q's receive buffer mapped into this process (NVLink peer memory); the pass stores every
    // output row straight into its receiver and d_out is not touched.
    static void slab_pass(const gpu_t& gpu, int which, const T* d_in, T* d_out, uint32_t lg_n,
                          uint32_t lg_g, uint32_t rank, Direction direction, cudaStream_t stream,
                          void* const* peers = nullptr)
    {
        const bool inverse = direction == Direction::inverse;
        if (lg_n > (uint32_t)F::MAX_LG || lg_n > 30 || rank >= (1u << lg_g))
            throw cuda_error(-(int)cudaErrorInvalidValue, "NTT slab: bad lg_domain_size / rank");
        const uint32_t lg_local = lg_n - lg_g;
        SlabPlan sp;
        if (!make_slab_plan(sp, lg_n, lg_g, rank, inverse, block_lg_tile(lg_local, 1, FieldId<F>::lg_tile), F::NTT_MAX_LG_R))
            throw cuda_error(-(int)cudaErrorInvalidValue,
                             "NTT slab: the first digit of lg_domain_size and the rest must both be >= lg_g");
        if (which == 2 && sp.needs_scratch && d_out == d_in)
            throw cuda_error(-(int)cudaErrorInvalidValue, "NTT slab: this size needs a scratch buffer distinct from the data");
        const Tables<F>& tb = tables(gpu, lg_n, inverse, stream);
        smem_opt_in<pass_kernel<F>>(gpu.cid(), (int)gpu.props().sharedMemPerBlockOptin);
        g_profile.reset();
        auto run = [&](const Pass& d, const T* src, T* dst) {
            uint32_t ntiles = 1u << (lg_local - d.lg_r - d.lg_w);
            size_t smem = smem_elems(d) * sizeof(T);
            g_profile.mark("pass", stream);
            if (!launch_static<F>(d, tb, src, dst, ntiles, smem, stream))
                pass_kernel<F><<<ntiles, tile_threads<F>(d), smem, stream>>>(d, tb, src, dst);
            COUNT_LAUNCH();
            CUDA_OK(cudaGetLastError());
        };
        if (which == 1 && peers != nullptr) {
            if (lg_g > 3)
                throw cuda_error(-(int)cudaErrorInvalidValue, "NTT slab: fused exchange supports up to 8 ranks");
            Pass d = sp.pass1;
            d.peer_on = 1;
            for (uint32_t q = 0; q < (1u << lg_g); q++) d.peer[q] = (uint64_t)(uintptr_t)peers[q];
            run(d, d_in, nullptr);
        } else if (which == 1) {
            run(sp.pass1, d_in, d_out);
        } else {
            T* buf[2] = {const_cast<T*>(d_in), d_out};
            for (const Pass& d : sp.after) run(d, buf[d.src], buf[d.dst]);
        }
        g_profile.mark("end", stream);
    }

    // Low-degree extension (reference: NTT::LDE / LDE_aux, ntt/ntt.cuh:247-340): `inout` holds
    // 2^lg_n evaluations on the size-2^lg_n domain and has room for 2^(lg_n+lg_blowup) elements;
    // on return it holds the evaluations of the same polynomial on the coset g*<w_ext> of the
    // extended domain, natural order.  aux_out (optional, 2^lg_n elements) receives the
    // polynomial's coefficients in natural order, as LDE_aux does.
    static RustError LDE(const gpu_t& gpu, T* inout, uint32_t lg_n, uint32_t lg_blowup, T* aux_out = nullptr)
    {
        const uint32_t lg_ext = lg_n + lg_blowup;
        if (lg_n == 0 || lg_ext > (uint32_t)F::MAX_LG || lg_ext > 30)
            return rust_err(-(int)cudaErrorInvalidValue, "LDE: lg_domain_size + lg_blowup out of range for this field");
        try {
            gpu.select();
            const stream_t& s = gpu[0];
            const size_t n = (size_t)1 << lg_n, n_ext = (size_t)1 << lg_ext;
            dev_ptr_t<T> d_in(n, s), d_ext(n_ext, s);
            s.HtoD(d_in, inout, n * sizeof(T));
            LDE_batch_dev(gpu, s, d_ext, d_in, lg_n, lg_blowup, 1);
            if (aux_out) {
                // natural-order coefficients = the bit-reversal of the NR inverse transform that
                // LDE_batch_dev leaves in d_in (the reference: bit_rev(aux_data, domain_data),
                // ntt/ntt.cuh:312-315)
                dev_ptr_t<T> d_aux(n, s);
                uint32_t bl = (uint32_t)std::min<size_t>((n + 255) / 256, (size_t)gpu.sm_count() * 16);
                bitrev_copy_kernel<F><<<bl, 256, 0, s>>>(d_aux, d_in, lg_n);
                COUNT_LAUNCH();
                CUDA_OK(cudaGetLastError());
                s.DtoH(aux_out, d_aux, n * sizeof(T));
            }
            s.DtoH(inout, d_ext, n_ext * sizeof(T));
            s.sync();
        } catch (const cuda_error& e) {
            try { gpu.sync(); } catch (...) {}
            return rust_err(e.code(), e.what());
        }
        return rust_ok();
    }

    // NTT::LDE_powers (ntt/ntt.cuh:352-356): d_inout[i] *= group_gen^bitrev(i), device memory,
    // enqueued on `stream`
    static void LDE_powers(const gpu_t& gpu, cudaStream_t stream, T* d_inout, uint32_t lg_n)
    {
        if (lg_n > (uint32_t)F::MAX_LG || lg_n > 30)
            throw cuda_error(-(int)cudaErrorInvalidValue, "LDE_powers: lg_domain_size out of range");
        coset_scale(gpu, d_inout, lg_n, true, false, stream);
    }
    // NTT::LDE_expand (ntt/ntt.cuh:358-365): d_out[i << lg_blowup] = d_in[i], zero elsewhere, no
    // coset shift; d_in is in bit-reversed order and may be the tail of d_out (then it is moved
    // aside first: the reference reads everything before a grid-wide barrier, same effect)
    static void LDE_expand(const gpu_t& gpu, cudaStream_t stream, T* d_out, const T* d_in, uint32_t lg_n,
                           uint32_t lg_blowup)
    {
        const uint32_t lg_ext = lg_n + lg_blowup;
        if (lg_ext > (uint32_t)F::MAX_LG || lg_ext > 30)
            throw cuda_error(-(int)cudaErrorInvalidValue, "LDE_expand: lg_domain_size + lg_blowup out of range");
        const size_t n = (size_t)1 << lg_n, n_ext = (size_t)1 << lg_ext;
        const stream_t st(stream);
        const bool overlap = d_in < d_out + n_ext && d_out < d_in + n;
        std::unique_ptr<dev_ptr_t<T>> tmp;
        if (overlap) {
            tmp.reset(new dev_ptr_t<T>(n, st));
            CUDA_OK(cudaMemcpyAsync(tmp->get(), d_in, n * sizeof(T), cudaMemcpyDeviceToDevice, stream));
            d_in = tmp->get();
        }
        uint32_t blocks = (uint32_t)std::min<size_t>((n_ext + 255) / 256, (size_t)gpu.sm_count() * 16);
        lde_spread_kernel<F><<<blocks, 256, 0, stream>>>(d_out, d_in, lg_n, lg_blowup, nullptr, nullptr, nullptr, false);
        COUNT_LAUNCH();
        CUDA_OK(cudaGetLastError());
    }

    static void Base_dev_ptr(const gpu_t& gpu, cudaStream_t stream, T* d_inout, uint32_t lg_n,
                             InputOutputOrder order, Direction direction, Type type)
    {   NTT_internal(gpu, d_inout, lg_n, order, direction, type, stream);   }

    // rejects a batch whose byte size does not fit size_t (callers validate before any work)
    static bool batch_fits(uint32_t lg_n, size_t batch)
    {   return lg_n <= 30 && batch <= (SIZE_MAX / sizeof(T)) >> lg_n;   }

    // batched LDE on device memory, enqueued on `stream`: d_in holds `batch` rows of 2^lg_n
    // evaluations and is left holding each row's coefficients in bit-reversed order; d_out receives
    // `batch` rows of 2^(lg_n + lg_blowup) evaluations on the coset, natural order (row by row what
    // LDE returns)
    static void LDE_batch_dev(const gpu_t& gpu, cudaStream_t stream, T* d_out, T* d_in, uint32_t lg_n,
                              uint32_t lg_blowup, size_t batch)
    {
        if (lg_n > 30 || lg_blowup > 30)
            throw cuda_error(-(int)cudaErrorInvalidValue, "LDE: lg_domain_size + lg_blowup out of range for this field");
        const uint32_t lg_ext = lg_n + lg_blowup;
        if (lg_ext > (uint32_t)F::MAX_LG || lg_ext > 30 || !batch_fits(lg_ext, batch))
            throw cuda_error(-(int)cudaErrorInvalidValue, "LDE: lg_domain_size + lg_blowup out of range for this field");
        if (lg_n == 0 || batch == 0) return;
        // the spread reads every row of d_in while writing d_out: the two must not overlap
        const size_t n_in = batch << lg_n, n_out = batch << lg_ext;
        if (d_in < d_out + n_out && d_out < d_in + n_in)
            throw cuda_error(-(int)cudaErrorInvalidValue, "LDE batch: d_out overlaps d_in");
        NTT_internal(gpu, d_in, lg_n, InputOutputOrder::NR, Direction::inverse, Type::standard, stream, batch);
        const CosetTables& ct = coset_tables(gpu, false, stream);
        const size_t n_ext = batch << lg_ext;
        uint32_t blocks = (uint32_t)std::min<size_t>((n_ext + 255) / 256, (size_t)gpu.sm_count() * 16);
        lde_spread_kernel<F><<<blocks, 256, 0, stream>>>(d_out, d_in, lg_n, lg_blowup, ct.g0, ct.g1, ct.g2, true, batch);
        COUNT_LAUNCH();
        CUDA_OK(cudaGetLastError());
        NTT_internal(gpu, d_out, lg_ext, InputOutputOrder::RN, Direction::forward, Type::standard, stream, batch);
    }

    // batched host-pointer entry: `batch` rows of 2^lg_n elements in place, synchronised.  The rows
    // travel in groups of about GROUP_BYTES through up to three device buffers: while group g is
    // transformed on stream 0, group g + 1 is uploaded on stream 1 and group g - 1 downloaded on
    // stream 2 (copies overlap transforms for pinned or registered memory; pageable memory goes
    // through the pinned staging ring, as in Base)
    static constexpr size_t GROUP_BYTES = (size_t)32 << 20;
    static RustError Base_batch(const gpu_t& gpu, T* inout, uint32_t lg_n, size_t batch, InputOutputOrder order,
                                Direction direction, Type type)
    {
        if (lg_n > (uint32_t)F::MAX_LG || lg_n > 30 || !batch_fits(lg_n, batch))   // before touching the buffer
            return rust_err(-(int)cudaErrorInvalidValue, "NTT batch: lg_domain_size or batch out of range for this field");
        if (lg_n == 0 || batch == 0) return rust_ok();
        const size_t row_bytes = sizeof(T) << lg_n;
        const size_t rows = std::min(batch, std::max<size_t>(1, GROUP_BYTES / row_bytes));
        // three buffers keep upload, transform and download all busy; groups of a GiB or more (one
        // huge row) make do with two.  Two or more buffers whenever there are two or more groups:
        // the upload of group g waits for the download of group g - nbuf, enqueued one step earlier
        const size_t ngroups = (batch + rows - 1) / rows;
        const size_t nbuf = std::min<size_t>(ngroups, rows * row_bytes >= ((size_t)1 << 30) ? 2 : 3);
        T* dbuf = nullptr;
        RustError result = rust_ok();
        try {
            gpu.select();
            const stream_t &comp = gpu[0], &up = gpu[1], &down = gpu[2];
            const bool pageable = batch * row_bytes >= ((size_t)8 << 20) && stager_t::is_pageable(inout);
            std::unique_lock<std::mutex> stage_lock(gpu.stage_mtx, std::defer_lock);
            if (pageable) stage_lock.lock();
            CUDA_OK(cudaMallocAsync((void**)&dbuf, nbuf * rows * row_bytes, comp));
            event_t allocated, uploaded[3], computed[3], downloaded[3];
            allocated.record(comp);
            allocated.wait(up);
            auto group = [&](size_t g, T*& dev, T*& host, size_t& bytes) {
                dev = dbuf + (g % nbuf) * (rows << lg_n);
                host = inout + ((g * rows) << lg_n);
                bytes = std::min(rows, batch - g * rows) * row_bytes;
            };
            // step i: upload + transform group i, then download group i - 1, so that a host-blocking
            // (pageable) copy of one group runs while the neighbouring group is being transformed
            for (size_t i = 0; i <= ngroups; i++) {
                T *dev, *host;
                size_t bytes;
                if (i < ngroups) {
                    group(i, dev, host, bytes);
                    const size_t b = i % nbuf;
                    if (i >= nbuf) downloaded[b].wait(up);        // buffer b's previous group has left
                    if (pageable) gpu.stager().HtoD(up, dev, host, bytes);
                    else up.HtoD(dev, host, bytes);
                    uploaded[b].record(up);
                    uploaded[b].wait(comp);
                    NTT_internal(gpu, dev, lg_n, order, direction, type, comp, bytes / row_bytes);
                    computed[b].record(comp);
                }
                if (i >= 1) {
                    group(i - 1, dev, host, bytes);
                    const size_t b = (i - 1) % nbuf;
                    computed[b].wait(down);
                    if (pageable) gpu.stager().DtoH(down, host, dev, bytes);
                    else down.DtoH(host, dev, bytes);
                    downloaded[b].record(down);
                }
            }
            downloaded[(ngroups - 1) % nbuf].wait(comp);
            CUDA_OK(cudaFreeAsync(dbuf, comp));
            dbuf = nullptr;
            gpu.sync();
        } catch (const cuda_error& e) {
            result = rust_err(e.code(), e.what());
        }
        if (dbuf) {
            try { gpu.sync(); } catch (...) {}
            (void)cudaFreeAsync(dbuf, gpu[0]);
        }
        return result;
    }

    // host-pointer entry: alloc + HtoD + transform + DtoH + sync, errors -> RustError
    static RustError Base(const gpu_t& gpu, T* inout, uint32_t lg_n, InputOutputOrder order,
                          Direction direction, Type type)
    {
        if (lg_n == 0) return rust_ok();
        if (lg_n > (uint32_t)F::MAX_LG || lg_n > 30)          // before touching the caller's buffer
            return rust_err(-(int)cudaErrorInvalidValue, "NTT: lg_domain_size out of range for this field");
        return host_round_trip(gpu, inout, (size_t)1 << lg_n, [&](T* d_inout, const stream_t& s) {
            NTT_internal(gpu, d_inout, lg_n, order, direction, type, s);
        });
    }

private:
    // n elements of host memory in place, synchronised, on stream 0: upload, transform(d_inout, stream)
    // on the device, download.  Pageable buffers (what the reference's Rust / Go callers pass) are
    // staged through pinned memory by worker threads; registered buffers go straight to the copy engine
    template<class Transform>
    static RustError host_round_trip(const gpu_t& gpu, T* inout, size_t n, Transform&& transform)
    {
        try {
            gpu.select();
            const stream_t& s = gpu[0];
            dev_ptr_t<T> d_inout(n, s);
            const bool pageable = n * sizeof(T) >= ((size_t)8 << 20) && stager_t::is_pageable(inout);
            std::unique_lock<std::mutex> stage_lock(gpu.stage_mtx, std::defer_lock);
            if (pageable) {
                stage_lock.lock();
                gpu.stager().HtoD(s, d_inout, inout, n * sizeof(T));
            } else {
                s.HtoD(d_inout, inout, n * sizeof(T));
            }
            transform(d_inout.get(), s);
            if (pageable) gpu.stager().DtoH(s, inout, d_inout, n * sizeof(T));
            else s.DtoH(inout, d_inout, n * sizeof(T));
            s.sync();
        } catch (const cuda_error& e) {
            try { gpu.sync(); } catch (...) {}
            return rust_err(e.code(), e.what());
        }
        return rust_ok();
    }
};

// NTT and LDE down the columns of a row-major 2^lg_n x width matrix, element (i, c) at word
// i * width + c, single-word fields.  Column c of the result is what NTT::NTT_internal returns for
// column c alone (same order, direction and type, the same coset exponents), without a transpose:
// the passes of the single-transform plan read and write tiles of adjacent matrix columns
// (set_matrix, matrix_pass_kernel).
template<class F>
struct NTTMatrix {
    typedef typename F::T T;
    typedef NTT<F> N;

    // rejects a matrix whose byte size does not fit size_t (callers validate before any work)
    static bool fits(uint32_t lg_n, size_t width)
    {   return lg_n <= 30 && width <= (SIZE_MAX / sizeof(T)) >> lg_n;   }

    // Tile shape, from the shape alone.  Every pass's sub-NTT is a digit of the single-transform plan
    // (2^12 rows at most, two passes up to 2^24); next to it, as many adjacent matrix columns as fill
    // a 2^14-element tile (the pass kernels' shared-memory tile), up to 64 and no more than the
    // width.  At 2^24 that is 4 columns, 32-byte row chunks for Goldilocks and 16-byte ones for
    // BabyBear; three passes of 2^8 rows with 16 columns were 15 % (Goldilocks) and 16 % (BabyBear)
    // slower on H100 at 2^24 x 16: the third pass costs more than the narrow chunks.  Below 2^22
    // elements in all the tile shrinks so that there are still >= 256 of them for the 132 SMs, as
    // for the batched passes.  DESIGN.md section 4.6 has the measurements.
    static uint32_t lg_tile(uint32_t lg_n, size_t width)
    {   return block_lg_tile(lg_n, width, FieldId<F>::lg_tile);   }

    static void coset_scale(const gpu_t& gpu, T* d, uint32_t lg_n, size_t width, bool bitrev, bool inverse,
                            cudaStream_t stream)
    {
        const auto& ct = N::coset_tables(gpu, inverse, stream);
        uint32_t bx = 1;
        while (bx < 256 && bx < width) bx <<= 1;
        const dim3 block(bx, 256 / bx);
        const size_t blocks = (((size_t)1 << lg_n) + block.y - 1) / block.y, cap = (size_t)gpu.sm_count() * 8;
        coset_matrix_kernel<F><<<(uint32_t)(blocks < cap ? blocks : cap), block, 0, stream>>>(d, lg_n, width, bitrev,
                                                                                         ct.g0, ct.g1, ct.g2);
        COUNT_LAUNCH();
        CUDA_OK(cudaGetLastError());
    }

    // device-resident, in place, enqueued on `stream`, no synchronisation
    static void transform(const gpu_t& gpu, T* d_inout, uint32_t lg_n, size_t width,
                          typename N::InputOutputOrder order, typename N::Direction direction,
                          typename N::Type type, cudaStream_t stream)
    {
        if (lg_n > (uint32_t)F::MAX_LG || !fits(lg_n, width))
            throw cuda_error(-(int)cudaErrorInvalidValue, "NTT matrix: lg_domain_size or width out of range for this field");
        if (lg_n == 0 || width == 0) return;
        const bool inverse = direction == N::Direction::inverse;
        const bool coset = type == N::Type::coset;
        // coset exponents as NTT_internal: bit-reversed for RR although the data is in natural order
        const bool in_rev = order != N::InputOutputOrder::NN && order != N::InputOutputOrder::NR;
        const bool out_rev = order != N::InputOutputOrder::NN && order != N::InputOutputOrder::RN;
        const uint32_t lg_t = lg_tile(lg_n, width);
        Plan plan = make_plan(lg_n, (int)order, inverse, lg_t, /*max_lg_w=*/0, F::NTT_MAX_LG_R);
        if (!set_matrix(plan, width, lg_t))
            throw cuda_error(-(int)cudaErrorInvalidValue, "NTT matrix: this plan has no matrix form");

        if (coset && !inverse) coset_scale(gpu, d_inout, lg_n, width, in_rev, false, stream);
        const Tables<F>& tb = N::tables(gpu, lg_n, inverse, stream);
        T* scratch = nullptr;
        if (plan.needs_scratch)
            CUDA_OK(cudaMallocAsync((void**)&scratch, (sizeof(T) * width) << lg_n, stream));
        T* buf[2] = {d_inout, scratch};
        g_profile.reset();
        for (const Pass& d : plan.passes) {
            g_profile.mark("pass", stream);
            launch_matrix<F>(d, tb, buf[d.src], buf[d.dst], width, lg_n, stream);
            COUNT_LAUNCH();
            CUDA_OK(cudaGetLastError());
        }
        g_profile.mark("end", stream);
        if (scratch) CUDA_OK(cudaFreeAsync(scratch, stream));
        if (coset && inverse) coset_scale(gpu, d_inout, lg_n, width, out_rev, true, stream);
    }

    // LDE of every column, enqueued on `stream`: d_in (2^lg_n x width evaluations) is left holding each
    // column's coefficients in bit-reversed row order; d_out receives 2^(lg_n + lg_blowup) x width
    // evaluations on the coset, natural order.  The same composition as NTT::LDE_batch_dev: inverse NR,
    // the spread with the coset shift, forward RN
    static void LDE_dev(const gpu_t& gpu, cudaStream_t stream, T* d_out, T* d_in, uint32_t lg_n, uint32_t lg_blowup,
                        size_t width)
    {
        if (lg_n > 30 || lg_blowup > 30)
            throw cuda_error(-(int)cudaErrorInvalidValue, "LDE matrix: lg_domain_size + lg_blowup out of range for this field");
        const uint32_t lg_ext = lg_n + lg_blowup;
        if (lg_ext > (uint32_t)F::MAX_LG || !fits(lg_ext, width))
            throw cuda_error(-(int)cudaErrorInvalidValue, "LDE matrix: lg_domain_size + lg_blowup out of range for this field");
        if (lg_n == 0 || width == 0) return;
        // the spread reads all of d_in while writing d_out: the two must not overlap
        const size_t n_in = width << lg_n, n_out = width << lg_ext;
        if (d_in < d_out + n_out && d_out < d_in + n_in)
            throw cuda_error(-(int)cudaErrorInvalidValue, "LDE matrix: d_out overlaps d_in");
        transform(gpu, d_in, lg_n, width, N::InputOutputOrder::NR, N::Direction::inverse, N::Type::standard, stream);
        const auto& ct = N::coset_tables(gpu, false, stream);
        uint32_t bx = 1;
        while (bx < 256 && bx < width) bx <<= 1;
        const dim3 block(bx, 256 / bx);
        const size_t blocks = (((size_t)1 << lg_ext) + block.y - 1) / block.y, cap = (size_t)gpu.sm_count() * 8;
        lde_spread_matrix_kernel<F><<<(uint32_t)(blocks < cap ? blocks : cap), block, 0, stream>>>(
            d_out, d_in, lg_n, lg_blowup, width, ct.g0, ct.g1, ct.g2);
        COUNT_LAUNCH();
        CUDA_OK(cudaGetLastError());
        transform(gpu, d_out, lg_ext, width, N::InputOutputOrder::RN, N::Direction::forward, N::Type::standard, stream);
    }

    // host memory, in place, synchronised: the whole matrix is uploaded, transformed and downloaded
    // (pageable memory through the pinned staging ring, as in NTT::Base)
    static RustError host(const gpu_t& gpu, T* inout, uint32_t lg_n, size_t width, typename N::InputOutputOrder order,
                          typename N::Direction direction, typename N::Type type)
    {
        if (lg_n > (uint32_t)F::MAX_LG || !fits(lg_n, width))       // before touching the caller's buffer
            return rust_err(-(int)cudaErrorInvalidValue, "NTT matrix: lg_domain_size or width out of range for this field");
        if (lg_n == 0 || width == 0) return rust_ok();
        return N::host_round_trip(gpu, inout, width << lg_n, [&](T* d_inout, const stream_t& s) {
            transform(gpu, d_inout, lg_n, width, order, direction, type, s);
        });
    }
};

}  // namespace ntt
