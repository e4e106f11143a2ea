// C-ABI entry points of the polynomial helpers (include/sppark_b200.h, "polynomial" block).
// Device pointers in, work enqueued on the caller's stream -- the calling convention of the
// reference's templates (polynomial/prefix_op.cuh:322, div_by_x_minus_z.cuh:445, evaluate.cuh:308),
// which take device arrays and a stream_t.
#include "../ff/field_dispatch.cuh"
#include "poly.cuh"

using namespace poly;

// scan shapes: E elements per thread, SBS threads per CTA.  The per-thread cost of carrying a scan
// across lanes and warps (ten joins) is amortised over E, so the wide fields, whose join is a
// 256-bit multiplication, take 8 per thread too and halve the CTA to keep the transpose buffer
// inside the static shared-memory limit.
template<class T> static constexpr int elems_per_thread() { return 8; }
template<class T> static constexpr int scan_threads() { return sizeof(T) >= 32 ? 128 : 256; }
static constexpr int BS = 256;                      // evaluate kernels

template<class F, int OP, int MODE, bool REV>
static uint32_t scan_capacity(const gpu_t& gpu)
{
    constexpr int E = elems_per_thread<typename F::T>(), SBS = scan_threads<typename F::T>();
    static int per_sm[64];                                   // occupancy per device, looked up once
    const int dev = gpu.cid() & 63;
    if (per_sm[dev] == 0) {
        int n = 0;
        CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, scan_kernel<F, OP, E, SBS, MODE, REV>, SBS, 0));
        per_sm[dev] = std::max(n, 1);
    }
    return (uint32_t)(gpu.sm_count() * per_sm[dev]);
}

template<class F, int OP, int MODE, bool REV>
static void scan_launch(const gpu_t& gpu, cudaStream_t stream, uint32_t grid_cap, typename F::T* out,
                        const typename F::T* in, size_t len,
                        const scan_tab<typename F::T, elems_per_thread<typename F::T>(), scan_threads<typename F::T>()>& z,
                        int rotate, uint32_t ntiles, typename F::T* aggs, typename F::T* edge)
{
    constexpr int E = elems_per_thread<typename F::T>(), SBS = scan_threads<typename F::T>();
    const uint32_t grid = std::min<uint32_t>(std::min<uint32_t>(ntiles, grid_cap), scan_capacity<F, OP, MODE, REV>(gpu));
    if (MODE == MODE_COOP) {
        void* args[] = {&out, &in, &len, (void*)&z, &rotate, &ntiles, &aggs, &edge};
        CUDA_OK(cudaLaunchCooperativeKernel((const void*)scan_kernel<F, OP, E, SBS, MODE, REV>, dim3(grid), dim3(SBS),
                                            args, 0, stream));
    } else {
        scan_kernel<F, OP, E, SBS, MODE, REV><<<grid, SBS, 0, stream>>>(out, in, len, z, rotate, ntiles, aggs, edge);
        CUDA_OK(cudaGetLastError());
    }
    COUNT_LAUNCH();
}

// a cooperative launch can be refused where an ordinary one is not (a device or a partition without
// cooperative-launch support, a grid the driver will not co-schedule): the plain launches still work
template<class Launch> static bool try_coop(Launch&& launch)
{
    try {
        launch();
        return true;
    } catch (const cuda_error& e) {
        if (e.code() == -(int)cudaErrorCooperativeLaunchTooLarge || e.code() == -(int)cudaErrorNotSupported ||
            e.code() == -(int)cudaErrorLaunchOutOfResources)
            return false;
        throw;
    }
}

template<class F, int OP>
static void scan(const gpu_t& gpu, cudaStream_t stream, typename F::T* out, const typename F::T* in, size_t len,
                 const typename F::T* z_host, int rotate)
{
    typedef typename F::T T;
    constexpr int E = elems_per_thread<T>(), SBS = scan_threads<T>();
    constexpr size_t TILE = (size_t)SBS * E;
    constexpr bool REV = OP == OP_DIV;
    if (len == 0) return;
    if (len > ((size_t)1 << 40)) throw cuda_error(-(int)cudaErrorInvalidValue, "polynomial: length out of range");
    const uint32_t ntiles = (uint32_t)((len + TILE - 1) / TILE);
    const stream_t st(stream);
    dev_ptr_t<T> scratch(2 * (size_t)ntiles + (ntiles + TILE - 1) / TILE, st);
    T* aggs = scratch.get();
    T* edge = aggs + ntiles;
    T* aggs2 = edge + ntiles;                                // aggregates of the aggregates' tiles
    scan_tab<T, E, SBS> zk{}, zt{};                          // powers of z; of z^TILE for the aggregates' scan
    if (OP == OP_DIV) {
        scan_tab_fill<F, E, SBS>(zk, arith<F>::konst(*z_host));
        scan_tab_fill<F, E, SBS>(zt, zk.zt);
    }
    bool parked = rotate != 0;                               // rotate: are boundary coefficients in edge[]?
    if (ntiles <= 2) {
        scan_launch<F, OP, MODE_SERIAL, REV>(gpu, stream, 1, out, in, len, zk, rotate, ntiles, aggs, edge);
    } else if (ntiles <= scan_capacity<F, OP, MODE_COOP, REV>(gpu) && !getenv("SPPARK_B200_POLY_NO_COOP") &&
               try_coop([&] { scan_launch<F, OP, MODE_COOP, REV>(gpu, stream, ~0u, out, in, len, zk, rotate, ntiles, aggs, edge); })) {
        parked = false;
    } else {
        const uint32_t rgrid = std::min<uint32_t>(ntiles, (uint32_t)gpu.sm_count() * 8);
        tile_reduce_kernel<F, OP, E, SBS><<<rgrid, SBS, 0, stream>>>(aggs, in, len, zk, REV, ntiles);
        COUNT_LAUNCH();
        CUDA_OK(cudaGetLastError());
        // the aggregates' own scan: a few tiles; one CTA walking them serially is a chain of ~25 dependent
        // joins per tile, so beyond two tiles they run side by side
        const uint32_t nagg_tiles = (uint32_t)((ntiles + TILE - 1) / TILE);
        if (!(nagg_tiles > 2 && nagg_tiles <= scan_capacity<F, OP, MODE_COOP, false>(gpu) &&
              try_coop([&] { scan_launch<F, OP, MODE_COOP, false>(gpu, stream, ~0u, aggs, aggs, ntiles, zt, 0, nagg_tiles, aggs2, nullptr); })))
            scan_launch<F, OP, MODE_SERIAL, false>(gpu, stream, 1, aggs, aggs, ntiles, zt, 0, nagg_tiles, nullptr, nullptr);
        scan_launch<F, OP, MODE_SCAN, REV>(gpu, stream, ~0u, out, in, len, zk, rotate, ntiles, aggs, edge);
    }
    if (OP == OP_DIV && parked && ntiles > 1) {
        scan_edge_kernel<T><<<(ntiles + 255) / 256, 256, 0, stream>>>(out, edge, len, ntiles, (uint32_t)TILE);
        COUNT_LAUNCH();
        CUDA_OK(cudaGetLastError());
    }
}

template<class F>
static void evaluate(const gpu_t& gpu, cudaStream_t stream, typename F::T* d_ret, const typename F::T* d_x, size_t n,
                     const typename F::T* d_coeffs, size_t len)
{
    typedef typename F::T T;
    if (n == 0) return;
    if (n > 0xffffffffu || len > ((size_t)1 << 40))
        throw cuda_error(-(int)cudaErrorInvalidValue, "evaluate: size out of range");
    // points that share one pass over the coefficients (accumulators in registers)
    constexpr int MAXPTS = sizeof(T) >= 32 ? 2 : 4;
    const int pts = n >= (size_t)MAXPTS ? MAXPTS : n >= 2 ? 2 : 1;
    auto kernel = pts == 4 ? evaluate_partial_kernel<F, BS, MAXPTS> :
                  pts == 2 ? evaluate_partial_kernel<F, BS, 2> : evaluate_partial_kernel<F, BS, 1>;
    int per_sm = 0;
    CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, BS, 0));
    // a resident grid, but at least 8 coefficients per thread before another CTA is worth its reduction;
    // short polynomials stay in ONE CTA, whose "partial" is the answer itself (one launch, no scratch)
    uint32_t nparts = (uint32_t)std::max<size_t>(1, std::min<size_t>((size_t)gpu.sm_count() * std::max(per_sm, 1),
                                                                    (len + (size_t)BS * 8 - 1) / ((size_t)BS * 8)));
    if (len <= ((size_t)1 << 14)) nparts = 1;
    if (nparts == 1) {
        kernel<<<1, BS, 0, stream>>>(d_ret, d_x, (uint32_t)n, d_coeffs, len);
        COUNT_LAUNCH();
        CUDA_OK(cudaGetLastError());
        return;
    }
    const stream_t st(stream);
    dev_ptr_t<T> partial((size_t)n * nparts, st);
    kernel<<<nparts, BS, 0, stream>>>(partial, d_x, (uint32_t)n, d_coeffs, len);
    COUNT_LAUNCH();
    CUDA_OK(cudaGetLastError());
    evaluate_finish_kernel<F, BS><<<(uint32_t)n, BS, 0, stream>>>(d_ret, partial, d_x, nparts, (uint32_t)BS);
    COUNT_LAUNCH();
    CUDA_OK(cudaGetLastError());
}

template<class F>
static void batch_inverse(const gpu_t& gpu, cudaStream_t stream, typename F::T* d_out, const typename F::T* d_inp,
                          size_t len)
{
    typedef typename F::T T;
    constexpr bool wide = sizeof(T) >= 32;
    constexpr int N = wide ? 4 : 8;
    constexpr int IBS = wide ? 512 : 256;
    if (len == 0) return;
    const size_t nchunks = (len + (size_t)IBS * N - 1) / ((size_t)IBS * N);
    const uint32_t grid = (uint32_t)std::min<size_t>(nchunks, (size_t)gpu.sm_count() * 8);
    // one inversion per chunk inside the kernel: always for the word fields (their inversion is ~100 short
    // multiplications; hoisting it measured slower on the GPU this was tuned on), and for the wide
    // fields while every chunk has an SM to itself
    if (!wide || nchunks <= 2 * (size_t)gpu.sm_count()) {
        batch_inverse_kernel<F, N, IBS, INV_SELF><<<grid, IBS, 0, stream>>>(d_out, d_inp, len, nullptr);
        COUNT_LAUNCH();
        CUDA_OK(cudaGetLastError());
        return;
    }
    const stream_t st(stream);
    dev_ptr_t<T> tots(nchunks, st);
    batch_inverse_kernel<F, N, IBS, INV_PRODUCT><<<grid, IBS, 0, stream>>>(nullptr, d_inp, len, tots);
    COUNT_LAUNCH();
    CUDA_OK(cudaGetLastError());
    batch_inverse<F>(gpu, stream, tots, tots, nchunks);      // chunk products are never zero
    batch_inverse_kernel<F, N, IBS, INV_GIVEN><<<grid, IBS, 0, stream>>>(d_out, d_inp, len, tots);
    COUNT_LAUNCH();
    CUDA_OK(cudaGetLastError());
}

enum { WHAT_PREFIX_ADD, WHAT_PREFIX_MUL, WHAT_DIV, WHAT_EVAL, WHAT_INV };

// every polynomial entry: the field's helper `what` on the caller's stream
static RustError run(int field, int what, void* a, const void* b, size_t n, const void* c, size_t len, int flag,
                     void* stream)
{
    return with_field(field, "sppark_b200 polynomial: unknown field", [&](auto t) {
        typedef typename decltype(t)::type F;
        typedef typename F::T T;
        return guarded([&] {
            const gpu_t& gpu = gpu_of_current_device();
            cudaStream_t s = (cudaStream_t)stream;
            switch (what) {
            case WHAT_PREFIX_ADD: scan<F, OP_ADD>(gpu, s, (T*)a, (const T*)b, len, nullptr, 0); break;
            case WHAT_PREFIX_MUL: scan<F, OP_MUL>(gpu, s, (T*)a, (const T*)b, len, nullptr, 0); break;
            case WHAT_DIV: scan<F, OP_DIV>(gpu, s, (T*)a, (const T*)a, len, (const T*)c, flag); break;
            case WHAT_EVAL: evaluate<F>(gpu, s, (T*)a, (const T*)b, n, (const T*)c, len); break;
            default: batch_inverse<F>(gpu, s, (T*)a, (const T*)b, len); break;
            }
            return rust_ok();
        });
    });
}

extern "C" RustError sppark_b200_prefix_op_dev(int field, int op, void* d_out, const void* d_inp, size_t len,
                                               void* stream)
{
    if (op != 0 && op != 1) return rust_err(-(int)cudaErrorInvalidValue, "sppark_b200_prefix_op_dev: op is 0 (add) or 1 (multiply)");
    return run(field, op == 0 ? WHAT_PREFIX_ADD : WHAT_PREFIX_MUL, d_out, d_inp, 0, nullptr, len, 0, stream);
}

extern "C" RustError sppark_b200_div_by_x_minus_z_dev(int field, void* d_inout, size_t len, const void* z,
                                                      int rotate, void* stream)
{
    if (z == nullptr) return rust_err(-(int)cudaErrorInvalidValue, "sppark_b200_div_by_x_minus_z_dev: z is null");
    return run(field, WHAT_DIV, d_inout, nullptr, 0, z, len, rotate != 0, stream);
}

extern "C" RustError sppark_b200_evaluate_dev(int field, void* d_ret, const void* d_x, size_t n,
                                              const void* d_coeffs, size_t len, void* stream)
{   return run(field, WHAT_EVAL, d_ret, d_x, n, d_coeffs, len, 0, stream);   }

extern "C" RustError sppark_b200_batch_inverse_dev(int field, void* d_out, const void* d_inp, size_t len,
                                                   void* stream)
{   return run(field, WHAT_INV, d_out, d_inp, 0, nullptr, len, 0, stream);   }
