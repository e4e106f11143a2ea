// Curve dispatch for the MSM entry points, drop-in and extended (include/sppark_b200.h).
#include "../util/gpu.cuh"
#include "curve_ops.cuh"
#include <cstring>
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
static const curve_ops* curve_of(int curve)
{   return curve < 0 || curve > SPPARK_CURVE_BLS12_377_G2 ? nullptr : CURVES[curve];   }

// the drop-in entry points of poc/msm-cuda: BLS12-381 host points, 32-byte scalars
//   mult_pippenger           poc/msm-cuda/cuda/pippenger.cu:20-25       G1, packed {X, Y} rows
//   mult_pippenger_inf       poc/msm-cuda/cuda/pippenger_inf.cu:28-34   G1, rows of ffi_affine_sz bytes
//   mult_pippenger_fp2_inf   poc/msm-cuda/cuda/pippenger_inf.cu:36-43   G2, rows of ffi_affine_sz bytes
// The _inf rows always carry the infinity flag after Y, so a stride with no room for it is refused.
extern "C" RustError mult_pippenger(void* out, const void* points, size_t npoints, const void* scalars)
{   return curve_bls12_381.host(out, points, npoints, scalars, 96, false, false, 32, 255);   }

extern "C" RustError mult_pippenger_inf(void* out, const void* points, size_t npoints,
                                        const void* scalars, size_t ffi_affine_sz)
{   return curve_bls12_381.host(out, points, npoints, scalars, ffi_affine_sz, true, false, 32, 255);   }

extern "C" RustError mult_pippenger_fp2_inf(void* out, const void* points, size_t npoints,
                                            const void* scalars, size_t ffi_affine_sz)
{   return curve_bls12_381_g2.host(out, points, npoints, scalars, ffi_affine_sz, true, false, 32, 255);   }

extern "C" RustError sppark_b200_generate_points_dev(int curve, void* d_out, size_t n, void* stream)
{
    if (n >= (1ull << 31)) return rust_err(-(int)cudaErrorInvalidValue, "generate_points: n too large");
    const curve_ops* c = curve_of(curve);
    if (c == nullptr) return rust_err(-(int)cudaErrorInvalidValue, "generate_points: unknown curve");
    return c->gen(d_out, n, stream);
}

extern "C" RustError sppark_b200_msm_combine(int curve, void* out, const void* partials, size_t count)
{
    const curve_ops* c = curve_of(curve);
    if (c == nullptr) return rust_err(-(int)cudaErrorInvalidValue, "msm_combine: unknown curve");
    return c->combine(out, partials, count);
}

// ffi_affine_sz: 0 = packed {X, Y}; larger than that = arkworks rows with an infinity flag after Y
static RustError msm_any(int curve, void* out, const void* points, size_t npoints, const void* scalars,
                         size_t ffi_affine_sz, bool mont, uint32_t scalar_bytes = 32, uint32_t nbits = 255)
{
    const curve_ops* c = curve_of(curve);
    if (c == nullptr) return rust_err(-(int)cudaErrorInvalidValue, "sppark_b200_msm: unknown curve");
    return c->host(out, points, npoints, scalars, ffi_affine_sz ? ffi_affine_sz : c->affine_bytes,
                   ffi_affine_sz > c->affine_bytes, mont, scalar_bytes, nbits);
}

// a refused call returns infinity, as a failed MSM does
static RustError refuse(void* out, size_t jacobian_bytes, const std::string& msg)
{
    if (out) memset(out, 0, jacobian_bytes);
    return rust_err(-(int)cudaErrorInvalidValue, msg);
}
// the scalar format of the _bits entries: 4, 8, 16 or 32 bytes, 1 <= nbits <= min(255, 8 * bytes);
// code 0 when it is one
static RustError check_scalar_format(const char* entry, const curve_ops* c, void* out, uint32_t scalar_bytes,
                                     uint32_t nbits)
{
    const bool width = scalar_bytes == 4 || scalar_bytes == 8 || scalar_bytes == 16 || scalar_bytes == 32;
    if (width && nbits >= 1 && nbits <= 255 && nbits <= 8 * scalar_bytes) return rust_ok();
    return refuse(out, c->jacobian_bytes, std::string(entry) + ": scalar_bytes must be 4, 8, 16 or 32 and "
                                                               "1 <= nbits <= min(255, 8 * scalar_bytes)");
}

extern "C" RustError sppark_b200_msm_bits(int curve, void* out, const void* points, size_t npoints,
                                          const void* scalars, size_t ffi_affine_sz, uint32_t scalar_bytes,
                                          uint32_t nbits)
{
    const curve_ops* c = curve_of(curve);
    if (c == nullptr) return rust_err(-(int)cudaErrorInvalidValue, "sppark_b200_msm_bits: unknown curve");
    const RustError e = check_scalar_format("sppark_b200_msm_bits", c, out, scalar_bytes, nbits);
    if (e.code != 0) return e;
    return msm_any(curve, out, points, npoints, scalars, ffi_affine_sz, false, scalar_bytes, nbits);
}

extern "C" RustError sppark_b200_msm(int curve, void* out, const void* points, size_t npoints,
                                     const void* scalars, size_t ffi_affine_sz)
{   return msm_any(curve, out, points, npoints, scalars, ffi_affine_sz, false);   }

extern "C" RustError sppark_b200_msm_ex(int curve, void* out, const void* points, size_t npoints,
                                        const void* scalars, size_t ffi_affine_sz, int scalars_mont)
{   return msm_any(curve, out, points, npoints, scalars, ffi_affine_sz, scalars_mont != 0);   }

extern "C" RustError sppark_b200_msm_dev(int curve, void* out, const void* d_points, size_t npoints,
                                         const void* d_scalars, void* stream)
{
    const curve_ops* c = curve_of(curve);
    if (c == nullptr) return rust_err(-(int)cudaErrorInvalidValue, "sppark_b200_msm_dev: unknown curve");
    return c->dev(out, d_points, npoints, d_scalars, stream, 32, 255);
}

extern "C" RustError sppark_b200_msm_dev_bits(int curve, void* out, const void* d_points, size_t npoints,
                                              const void* d_scalars, uint32_t scalar_bytes, uint32_t nbits,
                                              void* stream)
{
    const curve_ops* c = curve_of(curve);
    if (c == nullptr) return rust_err(-(int)cudaErrorInvalidValue, "sppark_b200_msm_dev_bits: unknown curve");
    const RustError e = check_scalar_format("sppark_b200_msm_dev_bits", c, out, scalar_bytes, nbits);
    if (e.code != 0) return e;
    if ((uintptr_t)d_scalars % (scalar_bytes < 16 ? scalar_bytes : 16) != 0)   // one aligned load per scalar
        return refuse(out, c->jacobian_bytes, "sppark_b200_msm_dev_bits: d_scalars must be aligned to "
                                              "min(scalar_bytes, 16) bytes");
    return c->dev(out, d_points, npoints, d_scalars, stream, scalar_bytes, nbits);
}

// ---- one MSM sharded by point-chunk over several GPUs of this process (SURVEY.md section 8e) --------
// chunk i of the points / scalars runs on device_ids[i] (one host thread per distinct device, the
// chunks of a device one after the other; the host-pointer pipeline of msm_host on each device's
// own PCIe link), the partial results -- one Jacobian point each -- are added on the first device.
// No collective library is needed inside one process: the "all-gather" of the multi-process
// route (sppark_b200/parallel.py over NCCL) is a host array here.
extern "C" RustError sppark_b200_msm_sharded(int curve, void* out, const void* points, size_t npoints,
                                             const void* scalars, size_t ffi_affine_sz, int scalars_mont,
                                             const int* device_ids, size_t ndev)
{
    const curve_ops* c = curve_of(curve);
    if (c == nullptr) return rust_err(-(int)cudaErrorInvalidValue, "msm_sharded: unknown curve");
    if (out == nullptr || ndev == 0 || ndev > 64 || device_ids == nullptr)
        return rust_err(-(int)cudaErrorInvalidValue, "msm_sharded: need 1..64 device ids");
    const size_t jb = c->jacobian_bytes, stride = ffi_affine_sz ? ffi_affine_sz : c->affine_bytes;
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess) return rust_err(-(int)cudaErrorNoDevice, "msm_sharded: no CUDA device");
    for (size_t i = 0; i < ndev; i++)
        if (device_ids[i] < 0 || device_ids[i] >= count)
            return rust_err(-(int)cudaErrorInvalidDevice, "msm_sharded: no such device");
    int home = 0;
    (void)cudaGetDevice(&home);

    std::vector<uint8_t> partials(ndev * jb, 0);
    std::vector<RustError> status(ndev, rust_ok());
    const size_t chunk = (npoints + ndev - 1) / ndev;
    auto run_device = [&](int dev) {
        if (cudaSetDevice(dev) != cudaSuccess) {
            for (size_t i = 0; i < ndev; i++)
                if (device_ids[i] == dev) status[i] = rust_err(-(int)cudaErrorInvalidDevice, "msm_sharded: cudaSetDevice failed");
            return;
        }
        for (size_t i = 0; i < ndev; i++) {
            if (device_ids[i] != dev) continue;
            const size_t first = i * chunk < npoints ? i * chunk : npoints;
            const size_t n = npoints - first < chunk ? npoints - first : chunk;
            status[i] = msm_any(curve, partials.data() + i * jb, (const uint8_t*)points + first * stride, n,
                                (const uint8_t*)scalars + first * 32, ffi_affine_sz, scalars_mont != 0);
        }
    };
    std::vector<int> distinct;
    for (size_t i = 0; i < ndev; i++) {
        bool seen = false;
        for (int d : distinct) seen |= d == device_ids[i];
        if (!seen) distinct.push_back(device_ids[i]);
    }
    std::vector<std::thread> workers;
    for (size_t k = 1; k < distinct.size(); k++) workers.emplace_back(run_device, distinct[k]);
    run_device(distinct[0]);
    for (auto& t : workers) t.join();
    (void)cudaSetDevice(distinct[0]);
    RustError result = rust_ok();
    for (size_t i = 0; i < ndev; i++) {
        if (status[i].code != 0 && result.code == 0) result = status[i];
        else if (status[i].message) free(status[i].message);
    }
    if (result.code == 0) result = sppark_b200_msm_combine(curve, out, partials.data(), ndev);
    (void)cudaSetDevice(home);
    return result;
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
    if (out == nullptr) return rust_err(-(int)cudaErrorInvalidValue, "msm_ctx_create: null output");
    *out = nullptr;
    void* d = nullptr;
    const curve_ops* c = curve_of(curve);
    if (c == nullptr) return rust_err(-(int)cudaErrorInvalidValue, "msm_ctx_create: unknown curve");
    uint32_t wbits = 0;
    RustError e = c->preload(points, npoints, ffi_affine_sz ? ffi_affine_sz : c->affine_bytes,
                             ffi_affine_sz > c->affine_bytes, &d, &copies, &wbits);
    if (e.code != 0) return e;
    int dev = 0;
    (void)cudaGetDevice(&dev);
    *out = new sppark_b200_msm_ctx{curve, dev, d, npoints, copies, wbits};
    return rust_ok();
}

extern "C" RustError sppark_b200_msm_ctx_create(int curve, const void* points, size_t npoints,
                                                size_t ffi_affine_sz, sppark_b200_msm_ctx** out)
{   return ctx_create(curve, points, npoints, ffi_affine_sz, 1, out);   }

extern "C" RustError sppark_b200_msm_ctx_create_precomputed(int curve, const void* points, size_t npoints,
                                                            size_t ffi_affine_sz, uint32_t copies,
                                                            sppark_b200_msm_ctx** out)
{
    if (copies == 0) {
        if (out) *out = nullptr;
        return rust_err(-(int)cudaErrorInvalidValue, "msm_ctx_create_precomputed: copies must be >= 1");
    }
    return ctx_create(curve, points, npoints, ffi_affine_sz, copies, out);
}

// the body of both invoke entries; a null context counts as one without points
static RustError ctx_invoke(const char* entry, sppark_b200_msm_ctx* ctx, void* out, const void* scalars,
                            size_t npoints, bool mont, uint32_t scalar_bytes, uint32_t nbits)
{
    if (ctx == nullptr || npoints > ctx->npoints)
        return rust_err(-(int)cudaErrorInvalidValue, std::string(entry) + ": more scalars than preloaded points");
    int cur = 0;
    (void)cudaGetDevice(&cur);
    if (cur != ctx->device)
        return rust_err(-(int)cudaErrorInvalidDevice, std::string(entry) + ": the points live on another device");
    return curve_of(ctx->curve)->resident(out, ctx->d_points, npoints, scalars, mont, ctx->wbits, ctx->copies,
                                          ctx->npoints, scalar_bytes, nbits);
}

extern "C" RustError sppark_b200_msm_ctx_invoke(sppark_b200_msm_ctx* ctx, void* out, const void* scalars,
                                                size_t npoints, int scalars_mont)
{   return ctx_invoke("msm_ctx_invoke", ctx, out, scalars, npoints, scalars_mont != 0, 32, 255);   }

extern "C" RustError sppark_b200_msm_ctx_invoke_bits(sppark_b200_msm_ctx* ctx, void* out, const void* scalars,
                                                     size_t npoints, uint32_t scalar_bytes, uint32_t nbits)
{
    if (ctx == nullptr) return rust_err(-(int)cudaErrorInvalidValue, "msm_ctx_invoke_bits: null context");
    const RustError e = check_scalar_format("msm_ctx_invoke_bits", curve_of(ctx->curve), out, scalar_bytes, nbits);
    if (e.code != 0) return e;
    return ctx_invoke("msm_ctx_invoke_bits", ctx, out, scalars, npoints, false, scalar_bytes, nbits);
}

// ---- batches: many scalar vectors against one point set -----------------------------------------
// A refusal sets all `batch` outputs to infinity, where their size is known and fits a size_t.
static RustError refuse_batch(void* out, size_t batch, size_t jacobian_bytes, const std::string& msg)
{
    if (out && batch <= SIZE_MAX / jacobian_bytes) memset(out, 0, batch * jacobian_bytes);
    return rust_err(-(int)cudaErrorInvalidValue, msg);
}

// the checks of both batch entries, before any device work; code 0 and *done = false when the call goes on
static RustError check_batch(const char* entry, const curve_ops* c, void* out, size_t npoints, size_t batch,
                             uint32_t scalar_bytes, uint32_t nbits, bool* done)
{
    *done = true;
    const std::string e(entry);
    const RustError f = check_scalar_format(entry, c, nullptr, scalar_bytes, nbits);
    if (f.code != 0) {
        if (out && batch <= SIZE_MAX / c->jacobian_bytes) memset(out, 0, batch * c->jacobian_bytes);
        return f;
    }
    if (batch > SIZE_MAX / c->jacobian_bytes || (npoints && batch > SIZE_MAX / npoints / scalar_bytes))
        return refuse_batch(out, batch, c->jacobian_bytes, e + ": batch * npoints * scalar_bytes overflows");
    if (batch == 0) return rust_ok();
    if (out == nullptr) return rust_err(-(int)cudaErrorInvalidValue, e + ": null output");
    *done = false;
    return rust_ok();
}

extern "C" RustError sppark_b200_msm_ctx_invoke_batch(sppark_b200_msm_ctx* ctx, void* out_jacobians,
                                                      const void* scalars, size_t npoints, size_t batch,
                                                      uint32_t scalar_bytes, uint32_t nbits)
{
    if (ctx == nullptr) return rust_err(-(int)cudaErrorInvalidValue, "msm_ctx_invoke_batch: null context");
    const curve_ops* c = curve_of(ctx->curve);
    bool done;
    const RustError e = check_batch("msm_ctx_invoke_batch", c, out_jacobians, npoints, batch, scalar_bytes, nbits, &done);
    if (e.code != 0 || done) return e;
    if (npoints > ctx->npoints)
        return refuse_batch(out_jacobians, batch, c->jacobian_bytes, "msm_ctx_invoke_batch: more scalars than preloaded points");
    int cur = 0;
    (void)cudaGetDevice(&cur);
    if (cur != ctx->device) {
        memset(out_jacobians, 0, batch * c->jacobian_bytes);
        return rust_err(-(int)cudaErrorInvalidDevice, "msm_ctx_invoke_batch: the points live on another device");
    }
    return c->resident_batch(out_jacobians, ctx->d_points, npoints, scalars, batch, false, ctx->wbits, ctx->copies,
                             ctx->npoints, scalar_bytes, nbits);
}

extern "C" RustError sppark_b200_msm_dev_batch(int curve, void* out_jacobians, const void* d_points, size_t npoints,
                                               const void* d_scalars, size_t batch, uint32_t scalar_bytes,
                                               uint32_t nbits, void* stream)
{
    const curve_ops* c = curve_of(curve);
    if (c == nullptr) return rust_err(-(int)cudaErrorInvalidValue, "sppark_b200_msm_dev_batch: unknown curve");
    bool done;
    const RustError e = check_batch("sppark_b200_msm_dev_batch", c, out_jacobians, npoints, batch, scalar_bytes, nbits,
                                    &done);
    if (e.code != 0 || done) return e;
    if ((uintptr_t)d_scalars % (scalar_bytes < 16 ? scalar_bytes : 16) != 0)   // one aligned load per scalar
        return refuse_batch(out_jacobians, batch, c->jacobian_bytes, "sppark_b200_msm_dev_batch: d_scalars must be "
                                                                     "aligned to min(scalar_bytes, 16) bytes");
    return c->dev_batch(out_jacobians, d_points, npoints, d_scalars, batch, stream, scalar_bytes, nbits);
}

// ---- scalar multiplication of point arrays: out[i] = s_i * P_i, packed affine rows ---------------
// Every refusal comes before any device work and leaves the output as it was.
static bool overlaps(const void* a, size_t a_bytes, const void* b, size_t b_bytes)
{
    const uintptr_t x = (uintptr_t)a, y = (uintptr_t)b;
    return x < y + b_bytes && y < x + a_bytes;
}

// the checks both entries share; code 0 and *done = false when the call goes on
static RustError check_scale(const char* entry, const curve_ops* c, void* out, const void* points, size_t npoints,
                             const void* scalars, size_t stride, uint32_t scalar_bytes, uint32_t nbits, bool* done)
{
    *done = true;
    const std::string e(entry);
    if (c == nullptr) return rust_err(-(int)cudaErrorInvalidValue, e + ": unknown curve");
    const RustError f = check_scalar_format(entry, c, nullptr, scalar_bytes, nbits);
    if (f.code != 0) return f;
    if (npoints == 0) return rust_ok();
    if (out == nullptr || points == nullptr || scalars == nullptr)
        return rust_err(-(int)cudaErrorInvalidValue, e + ": null pointer");
    if (npoints >= (1ull << 31)) return rust_err(-(int)cudaErrorInvalidValue, e + ": npoints must be < 2^31");
    const size_t out_bytes = npoints * c->affine_bytes;
    if ((overlaps(out, out_bytes, points, npoints * stride) && !(out == points && stride == c->affine_bytes)) ||
        overlaps(out, out_bytes, scalars, npoints * scalar_bytes))
        return rust_err(-(int)cudaErrorInvalidValue, e + ": the output may be the points (in place) but may not "
                                                         "overlap them or the scalars otherwise");
    *done = false;
    return rust_ok();
}

extern "C" RustError sppark_b200_scale_points_dev(int curve, void* d_out, const void* d_points, size_t npoints,
                                                  const void* d_scalars, uint32_t scalar_bytes, uint32_t nbits,
                                                  void* stream)
{
    const char* entry = "sppark_b200_scale_points_dev";
    const curve_ops* c = curve_of(curve);
    bool done;
    const RustError e = check_scale(entry, c, d_out, d_points, npoints, d_scalars, c ? c->affine_bytes : 0,
                                    scalar_bytes, nbits, &done);
    if (e.code != 0 || done) return e;
    if ((uintptr_t)d_scalars % (scalar_bytes < 16 ? scalar_bytes : 16) != 0)   // one aligned load per scalar
        return rust_err(-(int)cudaErrorInvalidValue, std::string(entry) + ": d_scalars must be aligned to "
                                                                          "min(scalar_bytes, 16) bytes");
    return c->scale_dev(d_out, d_points, npoints, d_scalars, scalar_bytes, nbits, stream);
}

extern "C" RustError sppark_b200_scale_points(int curve, void* out_affine, const void* points_affine, size_t npoints,
                                              const void* scalars, size_t ffi_affine_sz, uint32_t scalar_bytes,
                                              uint32_t nbits)
{
    const char* entry = "sppark_b200_scale_points";
    const curve_ops* c = curve_of(curve);
    const size_t stride = c == nullptr ? 0 : ffi_affine_sz ? ffi_affine_sz : c->affine_bytes;
    const bool has_flag = c != nullptr && ffi_affine_sz > c->affine_bytes;
    bool done;
    const RustError e = check_scale(entry, c, out_affine, points_affine, npoints, scalars, stride, scalar_bytes, nbits,
                                    &done);
    if (e.code != 0 || done) return e;
    if (stride < c->affine_bytes + (has_flag ? 1 : 0))
        return rust_err(-(int)cudaErrorInvalidValue, std::string(entry) + ": affine stride too small");
    if (stride % 4 != 0)                         // rows are packed on the device with 32-bit loads
        return rust_err(-(int)cudaErrorInvalidValue, std::string(entry) + ": affine stride must be a multiple of 4 bytes");
    return c->scale(out_affine, points_affine, npoints, scalars, stride, has_flag, scalar_bytes, nbits);
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
