// NTT instantiations and their C-ABI entry points (include/sppark_b200.h).
#include "../ff/field_dispatch.cuh"
#include "ntt.cuh"
#include <memory>
#include <vector>

namespace ntt {
// lg_tile: log2(elements) of one CTA's shared-memory tile: 128 KiB of data for either field
template<> struct FieldId<gl64> { static constexpr uint32_t id = 1, lg_tile = 14; };
template<> struct FieldId<bb31> { static constexpr uint32_t id = 2, lg_tile = 14; };
// 256-bit Montgomery scalar fields: 2^11-element tiles (64 KiB) + 64 KiB of sub-NTT twiddles
template<> struct FieldId<ff::bls12_381_fr_ntt> { static constexpr uint32_t id = 3, lg_tile = 11; };
template<> struct FieldId<ff::pallas_fr_ntt> { static constexpr uint32_t id = 4, lg_tile = 11; };
template<> struct FieldId<ff::vesta_fr_ntt> { static constexpr uint32_t id = 5, lg_tile = 11; };
template<> struct FieldId<ff::bn254_fr_ntt> { static constexpr uint32_t id = 6, lg_tile = 11; };
template<> struct FieldId<ff::bls12_377_fr_ntt> { static constexpr uint32_t id = 7, lg_tile = 11; };
// ---- statically shaped twins of the passes the planner emits for the common sizes ----------
// key = (lg_r, lg_w, in row-fast, out row-fast, in_rev, out_rev, tw_mode)
template<class F, uint32_t R, uint32_t W, bool IRF, bool ORF, bool IREV, bool OREV, uint32_t TW>
static bool try_static(const Pass& d, const Tables<F>& tb, const typename F::T* in, typename F::T* out,
                       uint32_t ntiles, size_t smem, cudaStream_t stream)
{
    if (d.lg_r != R || d.lg_w != W || (d.in_lg_sa == 0) != IRF || (d.out_lg_sa == 0) != ORF ||
        (d.in_rev != 0) != IREV || (d.out_rev != 0) != OREV || d.tw_mode != TW)
        return false;
    typedef KStat<R, W, IRF, ORF, IREV, OREV, TW> K;
    int dev = 0;
    CUDA_OK(cudaGetDevice(&dev));
    smem_opt_in<pass_kernel_static<F, K>>(dev, 226 * 1024);      // + the static mbarrier word <= 227 KiB
    // one CTA per SM (a tile fills the shared memory), each walking ntiles / grid tiles
    static int sms_of[64];
    if (!sms_of[dev & 63]) CUDA_OK(cudaDeviceGetAttribute(&sms_of[dev & 63], cudaDevAttrMultiProcessorCount, dev));
    const int sms = sms_of[dev & 63];
    uint32_t per_sm = smem <= 48 * 1024 ? 4 : smem <= 100 * 1024 ? 2 : 1;
    uint32_t grid = ntiles < (uint32_t)sms * per_sm ? ntiles : (uint32_t)sms * per_sm;
    pass_kernel_static<F, K><<<grid, tile_threads<F>(d), smem, stream>>>(d, tb, in, out, ntiles);
    return true;
}

// the seven (in-order, out-order, twiddle) combinations used by NN / NR / RN plans
template<class F, uint32_t R, uint32_t W>
static bool try_shapes(const Pass& d, const Tables<F>& tb, const typename F::T* in, typename F::T* out,
                       uint32_t ntiles, size_t smem, cudaStream_t stream)
{
    return try_static<F, R, W, false, true, false, false, TW_STORE>(d, tb, in, out, ntiles, smem, stream)    // NN first
        || try_static<F, R, W, false, false, false, false, TW_NONE>(d, tb, in, out, ntiles, smem, stream)    // NN last
        || try_static<F, R, W, false, false, false, false, TW_STORE>(d, tb, in, out, ntiles, smem, stream)   // NN middle
        || try_static<F, R, W, false, false, false, true, TW_STORE>(d, tb, in, out, ntiles, smem, stream)    // NR strided
        || try_static<F, R, W, true, true, false, true, TW_NONE>(d, tb, in, out, ntiles, smem, stream)       // NR last
        || try_static<F, R, W, true, true, true, false, TW_NONE>(d, tb, in, out, ntiles, smem, stream)       // RN first
        || try_static<F, R, W, false, false, true, false, TW_LOAD>(d, tb, in, out, ntiles, smem, stream);    // RN strided
}

template<class F> bool launch_static(const Pass& d, const Tables<F>& tb, const typename F::T* in,
                                     typename F::T* out, uint32_t ntiles, size_t smem, cudaStream_t stream)
{
    if (getenv("SPPARK_B200_NTT_GENERIC")) return false;
    // 256-bit fields run the run-time shaped kernel: static twins (shapes of 2^20, 2^22, 2^24) cost
    // a 9-minute compile of this translation unit for a small gain on the GPU this was tuned on;
    // the kernel's cost is elsewhere (DESIGN.md section 4.4)
    if constexpr (F::LG_EPT != 4) return false;
    else return try_shapes<F, 12, 2>(d, tb, in, out, ntiles, smem, stream)
        || try_shapes<F, 11, 3>(d, tb, in, out, ntiles, smem, stream)
        || try_shapes<F, 10, 4>(d, tb, in, out, ntiles, smem, stream)
        || try_shapes<F, 12, 1>(d, tb, in, out, ntiles, smem, stream)
        || try_shapes<F, 11, 2>(d, tb, in, out, ntiles, smem, stream)
        || try_shapes<F, 10, 3>(d, tb, in, out, ntiles, smem, stream)
        || try_shapes<F, 10, 2>(d, tb, in, out, ntiles, smem, stream)
        || try_shapes<F, 11, 1>(d, tb, in, out, ntiles, smem, stream)
        || try_shapes<F, 11, 0>(d, tb, in, out, ntiles, smem, stream)
        || try_shapes<F, 10, 1>(d, tb, in, out, ntiles, smem, stream)
        || try_shapes<F, 10, 0>(d, tb, in, out, ntiles, smem, stream)
        || try_shapes<F, 9, 5>(d, tb, in, out, ntiles, smem, stream);    // 2^27 = 9+9+9 (BabyBear's maximum)
}

// matrix passes: statically shaped kernels for the (lg_r, lg_w) tiles of the hot shapes (DESIGN.md
// section 4.6), one per shape for all orders (KShape); any other shape runs the run-time shaped one
template<class F, uint32_t R, uint32_t W>
static bool try_matrix(const Pass& d, const Tables<F>& tb, const typename F::T* in, typename F::T* out,
                       uint64_t width, uint32_t lg_n, cudaStream_t stream)
{
    if (d.lg_r != R || d.lg_w != W) return false;
    launch_matrix_pass<F, KShape<R, W>>(d, tb, in, out, width, lg_n, stream);
    return true;
}

template<class F> void launch_matrix(const Pass& d, const Tables<F>& tb, const typename F::T* in, typename F::T* out,
                                     uint64_t width, uint32_t lg_n, cudaStream_t stream)
{
    if (try_matrix<F, 12, 2>(d, tb, in, out, width, lg_n, stream)          // 2^24, 2^23
        || try_matrix<F, 11, 3>(d, tb, in, out, width, lg_n, stream)       // 2^22, 2^21
        || try_matrix<F, 10, 4>(d, tb, in, out, width, lg_n, stream)       // 2^20, width > 8
        || try_matrix<F, 10, 3>(d, tb, in, out, width, lg_n, stream)       // 2^20, width 5..8
        || try_matrix<F, 8, 4>(d, tb, in, out, width, lg_n, stream))       // 2^16, width > 8 (2^12-element tiles)
        return;
    launch_matrix_pass<F, KDyn>(d, tb, in, out, width, lg_n, stream);
}

template void launch_matrix<gl64>(const Pass&, const Tables<gl64>&, const uint64_t*, uint64_t*, uint64_t, uint32_t, cudaStream_t);
template void launch_matrix<bb31>(const Pass&, const Tables<bb31>&, const uint32_t*, uint32_t*, uint64_t, uint32_t, cudaStream_t);
template struct NTTMatrix<gl64>;
template struct NTTMatrix<bb31>;

template bool launch_static<gl64>(const Pass&, const Tables<gl64>&, const uint64_t*, uint64_t*, uint32_t, size_t, cudaStream_t);
template bool launch_static<bb31>(const Pass&, const Tables<bb31>&, const uint32_t*, uint32_t*, uint32_t, size_t, cudaStream_t);


template bool launch_static<ff::bls12_381_fr_ntt>(const Pass&, const Tables<ff::bls12_381_fr_ntt>&, const ff::bls12_381_fr_ntt::T*, ff::bls12_381_fr_ntt::T*, uint32_t, size_t, cudaStream_t);
template bool launch_static<ff::pallas_fr_ntt>(const Pass&, const Tables<ff::pallas_fr_ntt>&, const ff::pallas_fr_ntt::T*, ff::pallas_fr_ntt::T*, uint32_t, size_t, cudaStream_t);
template bool launch_static<ff::vesta_fr_ntt>(const Pass&, const Tables<ff::vesta_fr_ntt>&, const ff::vesta_fr_ntt::T*, ff::vesta_fr_ntt::T*, uint32_t, size_t, cudaStream_t);
template bool launch_static<ff::bn254_fr_ntt>(const Pass&, const Tables<ff::bn254_fr_ntt>&, const ff::bn254_fr_ntt::T*, ff::bn254_fr_ntt::T*, uint32_t, size_t, cudaStream_t);
template bool launch_static<ff::bls12_377_fr_ntt>(const Pass&, const Tables<ff::bls12_377_fr_ntt>&, const ff::bls12_377_fr_ntt::T*, ff::bls12_377_fr_ntt::T*, uint32_t, size_t, cudaStream_t);

template class NTT<gl64>;
template class NTT<bb31>;
template class NTT<ff::bls12_381_fr_ntt>;
template class NTT<ff::pallas_fr_ntt>;
template class NTT<ff::vesta_fr_ntt>;
template class NTT<ff::bn254_fr_ntt>;
template class NTT<ff::bls12_377_fr_ntt>;
}  // namespace ntt

// order 0..4 (NN, NR, RN, RR, BB), direction 0..1, type 0..1: anything else is refused, with the
// entry's own message, before any work
static bool bad_ntt_args(int order, int direction, int type)
{   return order < 0 || order > 4 || direction < 0 || direction > 1 || type < 0 || type > 1;   }

template<class F>
static RustError ntt_host(size_t device_id, void* inout, uint32_t lg, int order, int direction, int type)
{
    typedef ntt::NTT<F> N;
    if (bad_ntt_args(order, direction, type))
        return rust_err(-(int)cudaErrorInvalidValue, "compute_ntt: bad order/direction/type");
    return guarded([&] {
        return N::Base(select_gpu((int)device_id), (typename F::T*)inout, lg, (typename N::InputOutputOrder)order,
                       (typename N::Direction)direction, (typename N::Type)type);
    });
}

template<class F>
static RustError ntt_slab(int which, const void* d_in, void* d_out, uint32_t lg, uint32_t lg_g, uint32_t rank,
                          int direction, void* stream, void* const* peers = nullptr)
{
    typedef ntt::NTT<F> N;
    if (direction < 0 || direction > 1 || (which != 1 && which != 2))
        return rust_err(-(int)cudaErrorInvalidValue, "ntt_slab_pass: bad direction / pass");
    return guarded([&] {
        N::slab_pass(gpu_of_current_device(), which, (const typename F::T*)d_in, (typename F::T*)d_out, lg, lg_g,
                     rank, (typename N::Direction)direction, (cudaStream_t)stream, peers);
        return rust_ok();
    });
}

extern "C" RustError sppark_b200_lde_powers_dev(int field, void* d_inout, uint32_t lg, void* stream)
{
    return with_field(field, "sppark_b200_lde_*_dev: unknown field", [&](auto t) {
        typedef typename decltype(t)::type F;
        return guarded([&] {
            ntt::NTT<F>::LDE_powers(gpu_of_current_device(), (cudaStream_t)stream, (typename F::T*)d_inout, lg);
            return rust_ok();
        });
    });
}

extern "C" RustError sppark_b200_lde_expand_dev(int field, void* d_out, const void* d_in, uint32_t lg,
                                                uint32_t lg_blowup, void* stream)
{
    return with_field(field, "sppark_b200_lde_*_dev: unknown field", [&](auto t) {
        typedef typename decltype(t)::type F;
        return guarded([&] {
            ntt::NTT<F>::LDE_expand(gpu_of_current_device(), (cudaStream_t)stream, (typename F::T*)d_out,
                                    (const typename F::T*)d_in, lg, lg_blowup);
            return rust_ok();
        });
    });
}

extern "C" RustError sppark_b200_lde(int field, size_t device_id, void* inout, uint32_t lg, uint32_t lg_blowup, void* aux_out)
{
    return with_field(field, "sppark_b200_lde: unknown field", [&](auto t) {
        typedef typename decltype(t)::type F;
        return guarded([&] {
            return ntt::NTT<F>::LDE(select_gpu((int)device_id), (typename F::T*)inout, lg, lg_blowup,
                                    (typename F::T*)aux_out);
        });
    });
}

extern "C" RustError sppark_b200_ntt_slab_pass(int field, int which, const void* d_in, void* d_out,
                                               uint32_t lg, uint32_t lg_g, uint32_t rank, int direction, void* stream)
{
    return with_field(field, "sppark_b200_ntt_slab_pass: unknown field", [&](auto t) {
        return ntt_slab<typename decltype(t)::type>(which, d_in, d_out, lg, lg_g, rank, direction, stream);
    });
}

extern "C" RustError sppark_b200_ntt_slab_pass_p2p(int field, const void* d_in, void* const* peer_recv,
                                                   uint32_t lg, uint32_t lg_g, uint32_t rank, int direction, void* stream)
{
    if (peer_recv == nullptr) return rust_err(-(int)cudaErrorInvalidValue, "ntt_slab_pass_p2p: no peer buffers");
    return with_field(field, "sppark_b200_ntt_slab_pass_p2p: unknown field", [&](auto t) {
        return ntt_slab<typename decltype(t)::type>(1, d_in, nullptr, lg, lg_g, rank, direction, stream, peer_recv);
    });
}

// ---- one transform slab-sharded over several GPUs of THIS process (SURVEY.md section 8e) -----------
// Host array in natural order in and out (order NN).  Chunk r of the plan (ntt_plan.hpp:
// make_slab_plan) runs on device_ids[r]: strided upload of its column slab, local stage 1, the one
// exchange, local stage 2, strided download of its slab of the result.  The exchange is either
// fused into stage 1 -- every row is stored straight into the receiving GPU over NVLink, all devices
// being mapped into one address space by cudaDeviceEnablePeerAccess (no IPC handles inside one
// process) -- or, when the devices cannot see each other (or an id repeats: single-GPU tests),
// G^2 block copies (cudaMemcpyPeerAsync) between the staging and the receive buffers.  Ordering
// between devices is by events only; the host waits once, for the downloads.
template<class F>
static RustError ntt_sharded(void* inout, uint32_t lg, int direction, const int* ids, size_t ndev)
{
    typedef typename F::T T;
    typedef ntt::NTT<F> N;
    uint32_t lg_g = 0;
    while ((1u << lg_g) < ndev) lg_g++;
    if (ndev == 0 || (1u << lg_g) != ndev || lg_g > 3)
        return rust_err(-(int)cudaErrorInvalidValue, "ntt_sharded: 1, 2, 4 or 8 chunks");
    if (direction < 0 || direction > 1 || lg > (uint32_t)F::MAX_LG || lg > 30 || lg < 2 * lg_g || lg == 0)
        return rust_err(-(int)cudaErrorInvalidValue, "ntt_sharded: bad direction / lg_domain_size");
    int home = 0;
    (void)cudaGetDevice(&home);
    const uint32_t s1 = ntt::slab_first_digit(lg, F::NTT_MAX_LG_R), s2 = lg - s1;
    if (s1 < lg_g || s2 < lg_g) return rust_err(-(int)cudaErrorInvalidValue, "ntt_sharded: transform too small for this many chunks");
    const size_t n1 = (size_t)1 << s1, n2 = (size_t)1 << s2, G = ndev, c = n2 / G, dd = n1 / G;
    const size_t nloc = ((size_t)1 << lg) / G, blk = c * dd;
    std::vector<T*> d_in(G, nullptr), d_stage(G, nullptr), d_recv(G, nullptr);
    RustError result = rust_ok();
    try {
        bool distinct = true;
        for (size_t a = 0; a < G; a++)
            for (size_t b = a + 1; b < G; b++) distinct &= ids[a] != ids[b];
        bool fused = distinct && G > 1 && getenv("SPPARK_B200_NTT_EXCHANGE_COPY") == nullptr;
        for (size_t a = 0; a < G && fused; a++)
            for (size_t b = 0; b < G && fused; b++) {
                int ok = 0;
                if (a != b) { CUDA_OK(cudaDeviceCanAccessPeer(&ok, ids[a], ids[b])); fused &= ok != 0; }
            }
        std::vector<const gpu_t*> gpus(G);
        for (size_t r = 0; r < G; r++) gpus[r] = &select_gpu(ids[r]);
        std::vector<std::unique_ptr<event_t>> staged(G), landed(G);
        for (size_t r = 0; r < G; r++) {
            gpus[r]->select();
            if (fused)
                for (size_t q = 0; q < G; q++)
                    if (q != r) {
                        cudaError_t e = cudaDeviceEnablePeerAccess(ids[q], 0);
                        if (e == cudaErrorPeerAccessAlreadyEnabled) (void)cudaGetLastError();
                        else CUDA_OK(e);
                    }
            const stream_t& st = (*gpus[r])[0];
            // plain cudaMalloc: allocations of the stream-ordered pool are not visible to peers
            CUDA_OK(cudaMalloc((void**)&d_in[r], nloc * sizeof(T)));
            CUDA_OK(cudaMalloc((void**)&d_recv[r], nloc * sizeof(T)));
            if (!fused) CUDA_OK(cudaMalloc((void**)&d_stage[r], nloc * sizeof(T)));
            staged[r].reset(new event_t());
            landed[r].reset(new event_t());
            // column slab r of the [N1][N2] matrix -> dense [N1][N2/G]
            st.HtoD2D(d_in[r], c * sizeof(T), (const T*)inout + r * c, n2 * sizeof(T), c * sizeof(T), n1);
        }
        if (fused) {
            // receive buffers must exist before any peer writes into them
            for (size_t r = 0; r < G; r++) { gpus[r]->select(); landed[r]->record((*gpus[r])[0]); }
            std::vector<void*> peers(G);
            for (size_t q = 0; q < G; q++) peers[q] = d_recv[q];
            for (size_t r = 0; r < G; r++) {
                gpus[r]->select();
                const stream_t& st = (*gpus[r])[0];
                for (size_t q = 0; q < G; q++) if (q != r) landed[q]->wait(st);
                N::slab_pass(*gpus[r], 1, d_in[r], nullptr, lg, lg_g, (uint32_t)r, (typename N::Direction)direction, st, peers.data());
                staged[r]->record(st);
            }
        } else {
            for (size_t r = 0; r < G; r++) {
                gpus[r]->select();
                const stream_t& st = (*gpus[r])[0];
                N::slab_pass(*gpus[r], 1, d_in[r], d_stage[r], lg, lg_g, (uint32_t)r, (typename N::Direction)direction, st);
                staged[r]->record(st);
            }
            // block q of sender g's staging -> block g of receiver q, on the receiver's stream
            for (size_t q = 0; q < G; q++) {
                gpus[q]->select();
                const stream_t& st = (*gpus[q])[0];
                for (size_t g = 0; g < G; g++) {
                    staged[g]->wait(st);
                    if (ids[g] == ids[q])
                        CUDA_OK(cudaMemcpyAsync(d_recv[q] + g * blk, d_stage[g] + q * blk, blk * sizeof(T), cudaMemcpyDeviceToDevice, st));
                    else
                        CUDA_OK(cudaMemcpyPeerAsync(d_recv[q] + g * blk, ids[q], d_stage[g] + q * blk, ids[g], blk * sizeof(T), st));
                }
            }
        }
        for (size_t q = 0; q < G; q++) {
            gpus[q]->select();
            const stream_t& st = (*gpus[q])[0];
            if (fused) for (size_t g = 0; g < G; g++) if (g != q) staged[g]->wait(st);
            // the input slab is dead by now: it is the scratch of a multi-pass second stage
            N::slab_pass(*gpus[q], 2, d_recv[q], d_in[q], lg, lg_g, (uint32_t)q, (typename N::Direction)direction, st);
            // [N2][N1/G] -> columns q*N1/G.. of the [N2][N1] result, i.e. X[k1 + N1*k2]
            CUDA_OK(cudaMemcpy2DAsync((T*)inout + q * dd, n1 * sizeof(T), d_recv[q], dd * sizeof(T), dd * sizeof(T), n2,
                                      cudaMemcpyDeviceToHost, st));
        }
        for (size_t r = 0; r < G; r++) { gpus[r]->select(); (*gpus[r])[0].sync(); }
    } catch (const cuda_error& e) {
        result = rust_err(e.code(), e.what());
    } catch (const std::exception& e) {
        result = rust_err(-1, e.what());
    }
    for (size_t r = 0; r < G; r++) {
        if (cudaSetDevice(ids[r]) != cudaSuccess) continue;
        if (result.code != 0) (void)cudaDeviceSynchronize();
        (void)cudaFree(d_in[r]);
        (void)cudaFree(d_stage[r]);
        (void)cudaFree(d_recv[r]);
    }
    (void)cudaSetDevice(home);
    return result;
}

extern "C" RustError sppark_b200_ntt_sharded(int field, void* inout, uint32_t lg_domain_size, int ntt_direction,
                                             const int* device_ids, size_t ndev)
{
    if (inout == nullptr || device_ids == nullptr)
        return rust_err(-(int)cudaErrorInvalidValue, "ntt_sharded: null argument");
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess) return rust_err(-(int)cudaErrorNoDevice, "ntt_sharded: no CUDA device");
    for (size_t i = 0; i < ndev; i++)
        if (device_ids[i] < 0 || device_ids[i] >= count)
            return rust_err(-(int)cudaErrorInvalidDevice, "ntt_sharded: no such device");
    return with_field(field, "sppark_b200_ntt_sharded: unknown field", [&](auto t) {
        return ntt_sharded<typename decltype(t)::type>(inout, lg_domain_size, ntt_direction, device_ids, ndev);
    });
}

extern "C" RustError compute_ntt(size_t device_id, void* inout, uint32_t lg_domain_size,
                                 int ntt_order, int ntt_direction, int ntt_type)
{   return ntt_host<gl64>(device_id, inout, lg_domain_size, ntt_order, ntt_direction, ntt_type);   }

extern "C" RustError sppark_b200_ntt(int field, size_t device_id, void* inout, uint32_t lg,
                                     int order, int direction, int type)
{
    return with_field(field, "sppark_b200_ntt: unknown field", [&](auto t) {
        return ntt_host<typename decltype(t)::type>(device_id, inout, lg, order, direction, type);
    });
}

extern "C" RustError sppark_b200_ntt_dev(int field, void* d_inout, uint32_t lg, int order,
                                         int direction, int type, void* stream)
{
    return with_field(field, "sppark_b200_ntt_dev: unknown field", [&](auto t) {
        typedef typename decltype(t)::type F;
        typedef ntt::NTT<F> N;
        if (bad_ntt_args(order, direction, type))
            return rust_err(-(int)cudaErrorInvalidValue, "ntt_dev: bad order/direction/type");
        return guarded([&] {
            N::Base_dev_ptr(gpu_of_current_device(), (cudaStream_t)stream, (typename F::T*)d_inout, lg,
                            (typename N::InputOutputOrder)order, (typename N::Direction)direction,
                            (typename N::Type)type);
            return rust_ok();
        });
    });
}

extern "C" RustError sppark_b200_ntt_batch_dev(int field, void* d_inout, uint32_t lg, size_t batch, int order,
                                               int direction, int type, void* stream)
{
    return with_field(field, "sppark_b200_ntt_batch_dev: unknown field", [&](auto t) {
        typedef typename decltype(t)::type F;
        typedef ntt::NTT<F> N;
        if (bad_ntt_args(order, direction, type))
            return rust_err(-(int)cudaErrorInvalidValue, "ntt_batch_dev: bad order/direction/type");
        if (lg > (uint32_t)F::MAX_LG || !N::batch_fits(lg, batch))
            return rust_err(-(int)cudaErrorInvalidValue, "ntt_batch_dev: lg_domain_size or batch out of range for this field");
        return guarded([&] {
            N::NTT_internal(gpu_of_current_device(), (typename F::T*)d_inout, lg, (typename N::InputOutputOrder)order,
                            (typename N::Direction)direction, (typename N::Type)type, (cudaStream_t)stream, batch);
            return rust_ok();
        });
    });
}

extern "C" RustError sppark_b200_lde_batch_dev(int field, void* d_out, void* d_in, uint32_t lg, uint32_t lg_blowup,
                                               size_t batch, void* stream)
{
    return with_field(field, "sppark_b200_lde_batch_dev: unknown field", [&](auto t) {
        typedef typename decltype(t)::type F;
        return guarded([&] {
            ntt::NTT<F>::LDE_batch_dev(gpu_of_current_device(), (cudaStream_t)stream, (typename F::T*)d_out,
                                       (typename F::T*)d_in, lg, lg_blowup, batch);
            return rust_ok();
        });
    });
}

extern "C" RustError sppark_b200_ntt_batch(int field, size_t device_id, void* inout, uint32_t lg, size_t batch,
                                           int order, int direction, int type)
{
    return with_field(field, "sppark_b200_ntt_batch: unknown field", [&](auto t) {
        typedef typename decltype(t)::type F;
        typedef ntt::NTT<F> N;
        if (bad_ntt_args(order, direction, type))
            return rust_err(-(int)cudaErrorInvalidValue, "ntt_batch: bad order/direction/type");
        return guarded([&] {
            return N::Base_batch(select_gpu((int)device_id), (typename F::T*)inout, lg, batch,
                                 (typename N::InputOutputOrder)order, (typename N::Direction)direction,
                                 (typename N::Type)type);
        });
    });
}

// ---- NTT and LDE down the columns of a row-major matrix (ntt.cuh: NTTMatrix), Goldilocks and BabyBear ----
// an entry's refusals of an unknown field id and of a 256-bit field's id
#define MATRIX_REFUSALS(entry) \
    entry ": unknown field", entry ": the matrix entries serve Goldilocks and BabyBear only, not the 256-bit fields"

extern "C" RustError sppark_b200_ntt_matrix_dev(int field, void* d_inout, uint32_t lg, size_t width, int order,
                                                int direction, int type, void* stream)
{
    return with_word_field(field, MATRIX_REFUSALS("sppark_b200_ntt_matrix_dev"), [&](auto t) {
        typedef typename decltype(t)::type F;
        typedef ntt::NTT<F> N;
        if (bad_ntt_args(order, direction, type))
            return rust_err(-(int)cudaErrorInvalidValue, "ntt_matrix_dev: bad order/direction/type");
        if (lg > (uint32_t)F::MAX_LG || !ntt::NTTMatrix<F>::fits(lg, width))
            return rust_err(-(int)cudaErrorInvalidValue, "ntt_matrix_dev: lg_domain_size or width out of range for this field");
        return guarded([&] {
            ntt::NTTMatrix<F>::transform(gpu_of_current_device(), (typename F::T*)d_inout, lg, width,
                                         (typename N::InputOutputOrder)order, (typename N::Direction)direction,
                                         (typename N::Type)type, (cudaStream_t)stream);
            return rust_ok();
        });
    });
}

extern "C" RustError sppark_b200_lde_matrix_dev(int field, void* d_out, void* d_in, uint32_t lg, uint32_t lg_blowup,
                                                size_t width, void* stream)
{
    return with_word_field(field, MATRIX_REFUSALS("sppark_b200_lde_matrix_dev"), [&](auto t) {
        typedef typename decltype(t)::type F;
        return guarded([&] {
            ntt::NTTMatrix<F>::LDE_dev(gpu_of_current_device(), (cudaStream_t)stream, (typename F::T*)d_out,
                                       (typename F::T*)d_in, lg, lg_blowup, width);
            return rust_ok();
        });
    });
}

extern "C" RustError sppark_b200_ntt_matrix(int field, size_t device_id, void* inout, uint32_t lg, size_t width,
                                            int order, int direction, int type)
{
    return with_word_field(field, MATRIX_REFUSALS("sppark_b200_ntt_matrix"), [&](auto t) {
        typedef typename decltype(t)::type F;
        typedef ntt::NTT<F> N;
        if (bad_ntt_args(order, direction, type))
            return rust_err(-(int)cudaErrorInvalidValue, "ntt_matrix: bad order/direction/type");
        if (lg > (uint32_t)F::MAX_LG || !ntt::NTTMatrix<F>::fits(lg, width))
            return rust_err(-(int)cudaErrorInvalidValue, "ntt_matrix: lg_domain_size or width out of range for this field");
        if (lg == 0 || width == 0) return rust_ok();
        return guarded([&] {
            return ntt::NTTMatrix<F>::host(select_gpu((int)device_id), (typename F::T*)inout, lg, width,
                                           (typename N::InputOutputOrder)order, (typename N::Direction)direction,
                                           (typename N::Type)type);
        });
    });
}
