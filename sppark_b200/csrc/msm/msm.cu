// Curve dispatch and argument checks of the MSM entry points, drop-in and extended (include/sppark_b200.h).
// Every argument check is here, in the entries; the templates of msm_host.cuh take checked arguments.
// A refusal throws refusal(msg) inside the entry's guard, which returns it as -cudaErrorInvalidValue.
#include "../util/gpu.cuh"
#include "curve_ops.cuh"
#include <thread>
#include <vector>

// one row per curve id (curve_ops.cuh)
static const curve_ops* const CURVES[] = {
    &curve_bls12_381,       // SPPARK_CURVE_BLS12_381_G1
    &curve_pallas,          // SPPARK_CURVE_PALLAS
    &curve_vesta,           // SPPARK_CURVE_VESTA
    &curve_bls12_381_g2,    // SPPARK_CURVE_BLS12_381_G2
    &curve_bn254,           // SPPARK_CURVE_BN254_G1
    &curve_bls12_377,       // SPPARK_CURVE_BLS12_377_G1
    &curve_bn254_g2,        // SPPARK_CURVE_BN254_G2
    &curve_bls12_377_g2,    // SPPARK_CURVE_BLS12_377_G2
};
static_assert(sizeof(CURVES) / sizeof(CURVES[0]) == SPPARK_CURVE_BLS12_377_G2 + 1, "one row per curve id");

static cuda_error refusal(const std::string& msg) { return cuda_error(-(int)cudaErrorInvalidValue, msg); }

// the row of a curve id; any other id is refused with "<entry>: unknown curve"
static const curve_ops& curve_of(int curve, const std::string& entry)
{
    if (curve < 0 || curve > SPPARK_CURVE_BLS12_377_G2) throw refusal(entry + ": unknown curve");
    return *CURVES[curve];
}

// The guard of the entries that return Jacobian points: fn(c) under guarded(), where fn sets c to its
// curve's row once it knows it.  From then on the output's size is known, and every failure sets all
// `batch` outputs to infinity (where batch * jacobian_bytes fits a size_t), as the reference's
// out->inf() does.
template<class Fn> static RustError guarded_msm(void* out, size_t batch, Fn&& fn)
{
    const curve_ops* c = nullptr;
    const RustError e = guarded([&] { return fn(c); });
    if (e.code != 0 && c != nullptr && out != nullptr && batch <= SIZE_MAX / c->jacobian_bytes)
        memset(out, 0, batch * c->jacobian_bytes);
    return e;
}

// ---- the argument checks, one per rule ------------------------------------------------------------
// the scalar format of the _bits entries: 4, 8, 16 or 32 bytes, 1 <= nbits <= min(255, 8 * bytes)
static void check_format(const std::string& entry, uint32_t scalar_bytes, uint32_t nbits)
{
    const bool width = scalar_bytes == 4 || scalar_bytes == 8 || scalar_bytes == 16 || scalar_bytes == 32;
    if (!width || nbits < 1 || nbits > 255 || nbits > 8 * scalar_bytes)
        throw refusal(entry + ": scalar_bytes must be 4, 8, 16 or 32 and 1 <= nbits <= min(255, 8 * scalar_bytes)");
}

// device scalars are read with one aligned load each
static void check_dev_scalars(const std::string& entry, const void* d_scalars, uint32_t scalar_bytes)
{
    if ((uintptr_t)d_scalars % (scalar_bytes < 16 ? scalar_bytes : 16) != 0)
        throw refusal(entry + ": d_scalars must be aligned to min(scalar_bytes, 16) bytes");
}

// host rows: room for {X, Y} and the flag, and a multiple of 4 bytes (they are packed on the device
// with 32-bit loads)
static void check_rows(const std::string& entry, const curve_ops& c, const host_rows& rows)
{
    if (rows.stride < c.affine_bytes + (rows.has_flag ? 1 : 0)) throw refusal(entry + ": affine stride too small");
    if (rows.stride % 4 != 0) throw refusal(entry + ": affine stride must be a multiple of 4 bytes");
}

// a bucket entry keeps 31 bits of row index
static void check_npoints(const std::string& entry, size_t npoints)
{
    if (npoints >= (1ull << 31)) throw refusal(entry + ": npoints must be < 2^31");
}

static void check_table(size_t npoints, uint32_t copies)
{
    if ((uint64_t)copies * npoints >= (1ull << 31)) throw refusal("msm: copies * npoints must be < 2^31");
}

// ffi_affine_sz: 0 = packed {X, Y}; larger than that = arkworks rows with an infinity flag after Y
static host_rows rows_of(const curve_ops& c, const void* points, size_t ffi_affine_sz)
{   return {points, ffi_affine_sz ? ffi_affine_sz : c.affine_bytes, ffi_affine_sz > c.affine_bytes};   }

// ---- host points, host scalars ------------------------------------------------------------------
// the MSM of curve c over host rows: the size, then the stride (not for npoints == 0, a no-op that
// writes infinity), before the device lookup
static RustError host_msm(const curve_ops& c, void* out, const host_rows& rows, size_t npoints, const void* scalars,
                          bool mont, uint32_t scalar_bytes = 32, uint32_t nbits = 255)
{
    return guarded_msm(out, 1, [&](const curve_ops*& known) {
        known = &c;
        if (npoints != 0) {
            check_npoints("msm", npoints);
            check_rows("msm", c, rows);
        }
        c.msm(out, msm_points{rows}, npoints, scalars, 1, mont, scalar_bytes, nbits);
        return rust_ok();
    });
}

// the drop-in entry points of poc/msm-cuda: BLS12-381 host points, 32-byte scalars
//   mult_pippenger           poc/msm-cuda/cuda/pippenger.cu:20-25       G1, packed {X, Y} rows
//   mult_pippenger_inf       poc/msm-cuda/cuda/pippenger_inf.cu:28-34   G1, rows of ffi_affine_sz bytes
//   mult_pippenger_fp2_inf   poc/msm-cuda/cuda/pippenger_inf.cu:36-43   G2, rows of ffi_affine_sz bytes
// The _inf rows always carry the infinity flag after Y, so a stride with no room for it is refused.
extern "C" RustError mult_pippenger(void* out, const void* points, size_t npoints, const void* scalars)
{   return host_msm(curve_bls12_381, out, {points, 96, false}, npoints, scalars, false);   }

extern "C" RustError mult_pippenger_inf(void* out, const void* points, size_t npoints,
                                        const void* scalars, size_t ffi_affine_sz)
{   return host_msm(curve_bls12_381, out, {points, ffi_affine_sz, true}, npoints, scalars, false);   }

extern "C" RustError mult_pippenger_fp2_inf(void* out, const void* points, size_t npoints,
                                            const void* scalars, size_t ffi_affine_sz)
{   return host_msm(curve_bls12_381_g2, out, {points, ffi_affine_sz, true}, npoints, scalars, false);   }

static RustError msm_any(const char* entry, int curve, void* out, const void* points, size_t npoints,
                         const void* scalars, size_t ffi_affine_sz, bool mont, uint32_t scalar_bytes = 32,
                         uint32_t nbits = 255)
{
    return guarded_msm(out, 1, [&](const curve_ops*& c) {
        c = &curve_of(curve, entry);
        check_format(entry, scalar_bytes, nbits);
        return host_msm(*c, out, rows_of(*c, points, ffi_affine_sz), npoints, scalars, mont, scalar_bytes, nbits);
    });
}

extern "C" RustError sppark_b200_msm(int curve, void* out, const void* points, size_t npoints,
                                     const void* scalars, size_t ffi_affine_sz)
{   return msm_any("sppark_b200_msm", curve, out, points, npoints, scalars, ffi_affine_sz, false);   }

extern "C" RustError sppark_b200_msm_ex(int curve, void* out, const void* points, size_t npoints,
                                        const void* scalars, size_t ffi_affine_sz, int scalars_mont)
{   return msm_any("sppark_b200_msm", curve, out, points, npoints, scalars, ffi_affine_sz, scalars_mont != 0);   }

extern "C" RustError sppark_b200_msm_bits(int curve, void* out, const void* points, size_t npoints,
                                          const void* scalars, size_t ffi_affine_sz, uint32_t scalar_bytes,
                                          uint32_t nbits)
{
    return msm_any("sppark_b200_msm_bits", curve, out, points, npoints, scalars, ffi_affine_sz, false, scalar_bytes,
                   nbits);
}

// ---- one MSM sharded by point-chunk over several GPUs of this process (SURVEY.md section 8e) --------
// chunk i of the points / scalars runs on device_ids[i] (one host thread per distinct device, the
// chunks of a device one after the other; the host-pointer pipeline of msm_slices on each device's
// own PCIe link), the partial results -- one Jacobian point each -- are added on the first device.
// No collective library is needed inside one process: the "all-gather" of the multi-process
// route (sppark_b200/parallel.py over NCCL) is a host array here.
extern "C" RustError sppark_b200_msm_sharded(int curve, void* out, const void* points, size_t npoints,
                                             const void* scalars, size_t ffi_affine_sz, int scalars_mont,
                                             const int* device_ids, size_t ndev)
{
    return guarded_msm(out, 1, [&](const curve_ops*& known) {
        const curve_ops& c = curve_of(curve, "msm_sharded");
        known = &c;
        if (out == nullptr || ndev == 0 || ndev > 64 || device_ids == nullptr)
            throw refusal("msm_sharded: need 1..64 device ids");
        const host_rows rows = rows_of(c, points, ffi_affine_sz);
        const size_t jb = c.jacobian_bytes, chunk = (npoints + ndev - 1) / ndev;
        if (npoints != 0) {                     // the 2^31 limit is per chunk; chunk 0 is the largest
            check_npoints("msm", chunk);
            check_rows("msm", c, rows);
        }
        int count = 0;
        if (cudaGetDeviceCount(&count) != cudaSuccess) throw cuda_error(-(int)cudaErrorNoDevice, "msm_sharded: no CUDA device");
        for (size_t i = 0; i < ndev; i++)
            if (device_ids[i] < 0 || device_ids[i] >= count)
                throw cuda_error(-(int)cudaErrorInvalidDevice, "msm_sharded: no such device");
        int home = 0;
        (void)cudaGetDevice(&home);

        std::vector<uint8_t> partials(ndev * jb, 0);
        std::vector<RustError> status(ndev, rust_ok());
        auto run_device = [&](int dev) {
            const bool selected = cudaSetDevice(dev) == cudaSuccess;
            for (size_t i = 0; i < ndev; i++) {
                if (device_ids[i] != dev) continue;
                status[i] = guarded([&] {
                    if (!selected) throw cuda_error(-(int)cudaErrorInvalidDevice, "msm_sharded: cudaSetDevice failed");
                    const size_t first = i * chunk < npoints ? i * chunk : npoints;
                    const size_t n = npoints - first < chunk ? npoints - first : chunk;
                    const host_rows part{(const uint8_t*)rows.p + first * rows.stride, rows.stride, rows.has_flag};
                    c.msm(partials.data() + i * jb, msm_points{part}, n, (const uint8_t*)scalars + first * 32, 1,
                          scalars_mont != 0, 32, 255);
                    return rust_ok();
                });
            }
        };
        std::vector<int> distinct;
        for (size_t i = 0; i < ndev; i++) {
            bool seen = false;
            for (int d : distinct) seen |= d == device_ids[i];
            if (!seen) distinct.push_back(device_ids[i]);
        }
        {
            // joins the workers on every exit, also when starting one of them fails
            struct workers_t {
                std::vector<std::thread> t;
                ~workers_t() { for (auto& w : t) w.join(); }
            } workers;
            for (size_t k = 1; k < distinct.size(); k++) workers.t.emplace_back(run_device, distinct[k]);
            run_device(distinct[0]);
        }
        (void)cudaSetDevice(distinct[0]);
        RustError result = rust_ok();
        for (size_t i = 0; i < ndev; i++) {
            if (status[i].code != 0 && result.code == 0) result = status[i];
            else if (status[i].message) free(status[i].message);
        }
        if (result.code == 0) result = sppark_b200_msm_combine(curve, out, partials.data(), ndev);
        (void)cudaSetDevice(home);
        return result;
    });
}

extern "C" RustError sppark_b200_msm_combine(int curve, void* out, const void* partials, size_t count)
{
    return guarded_msm(out, 1, [&](const curve_ops*& c) {
        c = &curve_of(curve, "msm_combine");
        c->combine(out, partials, count);
        return rust_ok();
    });
}

// ---- preloaded points (the reference's msm_t{points, npoints} + invoke(out, scalars),
// msm/pippenger.cuh:377-390,582-601): the SRS stays on the device, only scalars cross PCIe ------
// copies > 1: d_points holds the precomputed table (csrc/msm/msm_table.cuh) of width wbits, `copies`
// copies of the npoints rows, copy-major
struct sppark_b200_msm_ctx {
    int curve, device;
    void* d_points;
    size_t npoints;
    uint32_t copies, wbits;
};

static RustError ctx_create(int curve, const void* points, size_t npoints, size_t ffi_affine_sz, uint32_t copies,
                            sppark_b200_msm_ctx** out)
{
    return guarded([&] {
        if (copies == 0) {
            if (out) *out = nullptr;
            throw refusal("msm_ctx_create_precomputed: copies must be >= 1");
        }
        if (out == nullptr) throw refusal("msm_ctx_create: null output");
        *out = nullptr;
        const curve_ops& c = curve_of(curve, "msm_ctx_create");
        const host_rows rows = rows_of(c, points, ffi_affine_sz);
        check_rows("msm", c, rows);
        check_npoints("msm", npoints);
        check_table(npoints, copies);
        // the context exists before its device buffer, so nothing can fail once that buffer is made
        std::unique_ptr<sppark_b200_msm_ctx> ctx(new sppark_b200_msm_ctx{curve, 0, nullptr, npoints, copies, 0});
        c.preload(rows, npoints, &ctx->d_points, &ctx->copies, &ctx->wbits);
        (void)cudaGetDevice(&ctx->device);
        *out = ctx.release();
        return rust_ok();
    });
}

extern "C" RustError sppark_b200_msm_ctx_create(int curve, const void* points, size_t npoints,
                                                size_t ffi_affine_sz, sppark_b200_msm_ctx** out)
{   return ctx_create(curve, points, npoints, ffi_affine_sz, 1, out);   }

extern "C" RustError sppark_b200_msm_ctx_create_precomputed(int curve, const void* points, size_t npoints,
                                                            size_t ffi_affine_sz, uint32_t copies,
                                                            sppark_b200_msm_ctx** out)
{   return ctx_create(curve, points, npoints, ffi_affine_sz, copies, out);   }

// the checks of both batch entries, after the format: false when there is nothing to do (batch == 0)
static bool check_batch(const std::string& entry, const curve_ops& c, void* out, size_t npoints, size_t batch,
                        uint32_t scalar_bytes)
{
    if (batch > SIZE_MAX / c.jacobian_bytes || (npoints && batch > SIZE_MAX / npoints / scalar_bytes))
        throw refusal(entry + ": batch * npoints * scalar_bytes overflows");
    if (batch == 0) return false;
    if (out == nullptr) throw refusal(entry + ": null output");
    return true;
}

// the body of the invoke entries, a null context refused with "<entry><if_null>": the context's
// MSM of `batch` vectors of npoints host scalars (`batched`: the batch entry, with its checks)
static RustError ctx_invoke(const std::string& entry, const char* if_null, sppark_b200_msm_ctx* ctx, void* out,
                            const void* scalars, size_t npoints, bool batched, size_t batch, bool mont,
                            uint32_t scalar_bytes, uint32_t nbits)
{
    return guarded_msm(out, batch, [&](const curve_ops*& c) {
        if (ctx == nullptr) throw refusal(entry + if_null);
        c = CURVES[ctx->curve];
        check_format(entry, scalar_bytes, nbits);
        if (batched && !check_batch(entry, *c, out, npoints, batch, scalar_bytes)) return rust_ok();
        if (npoints > ctx->npoints) throw refusal(entry + ": more scalars than preloaded points");
        int cur = 0;
        (void)cudaGetDevice(&cur);
        if (cur != ctx->device)
            throw cuda_error(-(int)cudaErrorInvalidDevice, entry + ": the points live on another device");
        c->msm(out, msm_points{{}, ctx->d_points, ctx->wbits, ctx->copies, ctx->npoints}, npoints, scalars, batch,
               mont, scalar_bytes, nbits);
        return rust_ok();
    });
}

// a null context counts as one without points
extern "C" RustError sppark_b200_msm_ctx_invoke(sppark_b200_msm_ctx* ctx, void* out, const void* scalars,
                                                size_t npoints, int scalars_mont)
{
    return ctx_invoke("msm_ctx_invoke", ": more scalars than preloaded points", ctx, out, scalars, npoints, false, 1,
                      scalars_mont != 0, 32, 255);
}

extern "C" RustError sppark_b200_msm_ctx_invoke_bits(sppark_b200_msm_ctx* ctx, void* out, const void* scalars,
                                                     size_t npoints, uint32_t scalar_bytes, uint32_t nbits)
{
    return ctx_invoke("msm_ctx_invoke_bits", ": null context", ctx, out, scalars, npoints, false, 1, false,
                      scalar_bytes, nbits);
}

extern "C" RustError sppark_b200_msm_ctx_invoke_batch(sppark_b200_msm_ctx* ctx, void* out_jacobians,
                                                      const void* scalars, size_t npoints, size_t batch,
                                                      uint32_t scalar_bytes, uint32_t nbits)
{
    return ctx_invoke("msm_ctx_invoke_batch", ": null context", ctx, out_jacobians, scalars, npoints, true, batch,
                      false, scalar_bytes, nbits);
}

extern "C" void sppark_b200_msm_ctx_free(sppark_b200_msm_ctx* ctx)
{
    if (ctx == nullptr) return;
    int cur = 0;
    (void)cudaGetDevice(&cur);
    if (cur != ctx->device) (void)cudaSetDevice(ctx->device);
    (void)cudaFree(ctx->d_points);
    if (cur != ctx->device) (void)cudaSetDevice(cur);
    delete ctx;
}

// ---- device points, device scalars ------------------------------------------------------------------
extern "C" RustError sppark_b200_msm_dev(int curve, void* out, const void* d_points, size_t npoints,
                                         const void* d_scalars, void* stream)
{
    return guarded_msm(out, 1, [&](const curve_ops*& c) {
        c = &curve_of(curve, "sppark_b200_msm_dev");
        c->dev(out, d_points, npoints, d_scalars, 1, stream, 32, 255);
        return rust_ok();
    });
}

extern "C" RustError sppark_b200_msm_dev_bits(int curve, void* out, const void* d_points, size_t npoints,
                                              const void* d_scalars, uint32_t scalar_bytes, uint32_t nbits,
                                              void* stream)
{
    const std::string entry = "sppark_b200_msm_dev_bits";
    return guarded_msm(out, 1, [&](const curve_ops*& c) {
        c = &curve_of(curve, entry);
        check_format(entry, scalar_bytes, nbits);
        check_dev_scalars(entry, d_scalars, scalar_bytes);
        c->dev(out, d_points, npoints, d_scalars, 1, stream, scalar_bytes, nbits);
        return rust_ok();
    });
}

extern "C" RustError sppark_b200_msm_dev_batch(int curve, void* out_jacobians, const void* d_points, size_t npoints,
                                               const void* d_scalars, size_t batch, uint32_t scalar_bytes,
                                               uint32_t nbits, void* stream)
{
    const std::string entry = "sppark_b200_msm_dev_batch";
    return guarded_msm(out_jacobians, batch, [&](const curve_ops*& c) {
        c = &curve_of(curve, entry);
        check_format(entry, scalar_bytes, nbits);
        if (!check_batch(entry, *c, out_jacobians, npoints, batch, scalar_bytes)) return rust_ok();
        check_dev_scalars(entry, d_scalars, scalar_bytes);
        c->dev(out_jacobians, d_points, npoints, d_scalars, batch, stream, scalar_bytes, nbits);
        return rust_ok();
    });
}

// ---- synthetic inputs ---------------------------------------------------------------------------------
extern "C" RustError sppark_b200_generate_points_dev(int curve, void* d_out, size_t n, void* stream)
{
    return guarded([&] {
        if (n >= (1ull << 31)) throw refusal("generate_points: n too large");
        curve_of(curve, "generate_points").gen(d_out, n, stream);
        return rust_ok();
    });
}

// ---- scalar multiplication of point arrays: out[i] = s_i * P_i, packed affine rows ---------------
// Every refusal comes before any device work and leaves the output as it was (plain guarded()).
static bool overlaps(const void* a, size_t a_bytes, const void* b, size_t b_bytes)
{
    const uintptr_t x = (uintptr_t)a, y = (uintptr_t)b;
    return x < y + b_bytes && y < x + a_bytes;
}

// the checks both entries share; false when there is nothing to do (npoints == 0)
static bool check_scale(const std::string& entry, const curve_ops& c, void* out, const void* points, size_t npoints,
                        const void* scalars, size_t stride, uint32_t scalar_bytes, uint32_t nbits)
{
    check_format(entry, scalar_bytes, nbits);
    if (npoints == 0) return false;
    if (out == nullptr || points == nullptr || scalars == nullptr) throw refusal(entry + ": null pointer");
    check_npoints(entry, npoints);
    const size_t out_bytes = npoints * c.affine_bytes;
    if ((overlaps(out, out_bytes, points, npoints * stride) && !(out == points && stride == c.affine_bytes)) ||
        overlaps(out, out_bytes, scalars, npoints * scalar_bytes))
        throw refusal(entry + ": the output may be the points (in place) but may not overlap them or the scalars "
                              "otherwise");
    return true;
}

extern "C" RustError sppark_b200_scale_points_dev(int curve, void* d_out, const void* d_points, size_t npoints,
                                                  const void* d_scalars, uint32_t scalar_bytes, uint32_t nbits,
                                                  void* stream)
{
    const std::string entry = "sppark_b200_scale_points_dev";
    return guarded([&] {
        const curve_ops& c = curve_of(curve, entry);
        if (!check_scale(entry, c, d_out, d_points, npoints, d_scalars, c.affine_bytes, scalar_bytes, nbits))
            return rust_ok();
        check_dev_scalars(entry, d_scalars, scalar_bytes);
        c.scale_dev(d_out, d_points, npoints, d_scalars, scalar_bytes, nbits, stream);
        return rust_ok();
    });
}

extern "C" RustError sppark_b200_scale_points(int curve, void* out_affine, const void* points_affine, size_t npoints,
                                              const void* scalars, size_t ffi_affine_sz, uint32_t scalar_bytes,
                                              uint32_t nbits)
{
    const std::string entry = "sppark_b200_scale_points";
    return guarded([&] {
        const curve_ops& c = curve_of(curve, entry);
        const host_rows rows = rows_of(c, points_affine, ffi_affine_sz);
        if (!check_scale(entry, c, out_affine, points_affine, npoints, scalars, rows.stride, scalar_bytes, nbits))
            return rust_ok();
        check_rows(entry, c, rows);
        c.scale(out_affine, rows, npoints, scalars, scalar_bytes, nbits);
        return rust_ok();
    });
}
