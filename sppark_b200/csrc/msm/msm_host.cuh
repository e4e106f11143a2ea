// MSM instantiations and their C-ABI entry points (include/sppark_b200.h).
//   mult_pippenger       poc/msm-cuda/cuda/pippenger.cu:20-25
//   mult_pippenger_inf   poc/msm-cuda/cuda/pippenger_inf.cu:28-34
// Host-pointer calls follow the reference's contract (msm/pippenger.cuh:730-747): scratch is
// allocated per call from the stream-ordered pool, scalars are 256-bit little-endian integers
// NOT in Montgomery form (mont=false), the result is a Jacobian point in Montgomery form.
#pragma once
#include "../ff/fields.cuh"
#include "msm.cuh"

namespace {

// Host-pointer MSM.  The points arrive over PCIe while the GPU is already accumulating: the
// input is cut into slices, slice k+1 is copied (copy stream, double-buffered) while slice k is
// sorted and folded into the persistent buckets (compute stream).  The reference overlaps the
// same way with its batches (msm/pippenger.cuh:505-557); here the bucket file is shared by all
// slices, so the running sums and the Horner pass run once at the end instead of once per batch.
// scalars handed over in Montgomery form (the reference's `mont = true`, the default of its C++
// mult_pippenger template, msm/pippenger.cuh:730-733; `breakdown` calls from() per scalar,
// :99-101): one Montgomery multiplication by 1 per scalar, in place on the device copy
template<class Fr>
__global__ void scalars_from_mont_kernel(uint32_t* scalars, size_t n)
{
    size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    Fr s, one;
#pragma unroll
    for (int k = 0; k < Fr::N; k++) { s.l[k] = scalars[i * Fr::N + k]; one.l[k] = k == 0; }
    s = s * one;
#pragma unroll
    for (int k = 0; k < Fr::N; k++) scalars[i * Fr::N + k] = s.l[k];
}
template<class Fr>
void scalars_from_mont(uint32_t* d_scalars, size_t n, cudaStream_t stream)
{
    scalars_from_mont_kernel<Fr><<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(d_scalars, n);
    COUNT_LAUNCH();
    CUDA_OK(cudaGetLastError());
}
typedef void (*unmont_fn)(uint32_t*, size_t, cudaStream_t);

// `resident` != nullptr: the points are already on the device as packed affine rows (preloaded by
// msm_preload below -- the reference's msm_t{points, npoints} constructor + invoke(out, scalars),
// msm/pippenger.cuh:377-390,582-601): only the scalars cross PCIe, sliced the same way.
template<class F>
RustError msm_host(void* out, const void* points, size_t npoints, const void* scalars,
                   size_t stride, bool has_flag, unmont_fn unmont = nullptr,
                   const uint32_t* resident = nullptr)
{
    constexpr size_t PB = 2 * F::N * 4, JB = 3 * F::N * 4;
    try {
        const gpu_t& gpu = select_gpu(-1);
        gpu.select();
        if (npoints == 0) { memset(out, 0, JB); return rust_ok(); }
        if (!resident && stride < PB + (has_flag ? 1 : 0))
            return rust_err(-(int)cudaErrorInvalidValue, "msm: affine stride too small");
        if (!resident && stride % 4 != 0)        // rows are packed on the device with 32-bit loads
            return rust_err(-(int)cudaErrorInvalidValue, "msm: affine stride must be a multiple of 4 bytes");
        const stream_t &compute = gpu[0], &copy = gpu[1];
        const bool packed = resident || (stride == PB && !has_flag);

        // slice schedule: a short first slice (the GPU idles while slice 0 crosses PCIe), then
        // doubling ones (fewer bucket reloads); slice k+1 is copied while slice k is computed
        std::vector<size_t> sched;
        if (const char* env = getenv("SPPARK_B200_MSM_SCHED")) {
            // experiments: relative slice sizes, e.g. "1,1,2,4,8"
            std::vector<size_t> w;
            size_t sum = 0;
            for (const char* p = env; *p;) {
                size_t v = strtoul(p, const_cast<char**>(&p), 10);
                if (v == 0) { w.clear(); break; }
                w.push_back(v);
                sum += v;
                if (*p == ',') p++;
            }
            size_t done = 0;
            for (size_t k = 0; k < w.size() && done < npoints; k++) {
                size_t part = k + 1 == w.size() ? npoints - done
                                                : std::min(npoints - done, ((npoints / sum * w[k]) + 31) & ~(size_t)31);
                if (part) sched.push_back(part);
                done += part;
            }
            if (sched.empty()) sched.push_back(npoints);
        } else if (const char* env = getenv("SPPARK_B200_MSM_SLICES")) {
            size_t k = std::max(1, atoi(env)), each = ((npoints + k - 1) / k + 31) & ~(size_t)31;
            for (size_t done = 0; done < npoints; done += each) sched.push_back(std::min(each, npoints - done));
        } else if (resident && npoints >= (1u << 22)) {
            // only 32 B per point cross PCIe: N/8 then the rest (chosen over N/4 + 3N/4, N/16 +
            // 15N/16 and the four-slice schedule below on an earlier GPU; not re-measured on H100)
            const size_t e = (npoints / 8 + 31) & ~(size_t)31;
            sched.push_back(e);
            sched.push_back(npoints - e);
        } else if (npoints >= (1u << 22)) {
            // N/16, N/8, N/4, 9N/16 (chosen over N/8, N/8, N/4, N/2 and five or six slices with
            // tools/probe_e2e.py on an earlier GPU; not re-measured on H100)
            const size_t e = (npoints / 16 + 31) & ~(size_t)31;
            for (size_t part : {e, 2 * e, 4 * e}) sched.push_back(part);
            sched.push_back(npoints - 7 * e);
        } else {
            sched.push_back(npoints);
        }
        const size_t nslices = sched.size(), nbuf = nslices > 1 ? 2 : 1;
        const size_t slice_n = *std::max_element(sched.begin(), sched.end());
        const bool pageable = (!resident && stager_t::is_pageable(points)) || stager_t::is_pageable(scalars);
        std::unique_lock<std::mutex> stage_lock(gpu.stage_mtx, std::defer_lock);
        if (pageable) stage_lock.lock();
        auto upload = [&](void* dst, const void* src, size_t bytes) {
            if (pageable) gpu.stager().HtoD(copy, dst, src, bytes);
            else copy.HtoD(dst, src, bytes);
        };

        dev_ptr_t<uint32_t> d_out(JB / 4, compute);
        dev_ptr_t<uint32_t> d_points(resident ? 1 : nbuf * slice_n * (PB / 4), compute), d_scalars(nbuf * slice_n * 8, compute);
        dev_ptr_t<uint8_t> d_raw(packed ? 1 : nbuf * slice_n * stride, compute);
        event_t copied[2], consumed[2], ready;
        ready.record(compute);                                    // buffers exist
        ready.wait(copy);

        // on any failure, drain both streams while the buffers above are still alive (their
        // stream-ordered frees run during unwinding)
        struct drain_t {
            const stream_t &a, &b;
            bool armed = true;
            ~drain_t() { if (armed) { (void)cudaStreamSynchronize(a); (void)cudaStreamSynchronize(b); } }
        } drain{compute, copy};

        msm::msm_t<F> m(gpu);
        auto job = m.begin(npoints, slice_n, compute);
        size_t first = 0;
        for (size_t k = 0; k < nslices; first += sched[k], k++) {
            const size_t b = k & (nbuf - 1), n = sched[k];
            const uint32_t* dp = resident ? resident + first * (PB / 4) : d_points + b * slice_n * (PB / 4);
            uint32_t* ds = d_scalars + b * slice_n * 8;
            if (k >= nbuf) consumed[b].wait(copy);                                // buffer free again
            upload(ds, (const uint8_t*)scalars + first * 32, n * 32);
            if (resident) {
            } else if (packed) {
                upload(d_points + b * slice_n * (PB / 4), (const uint8_t*)points + first * PB, n * PB);
            } else {
                uint8_t* dr = d_raw + b * slice_n * stride;
                upload(dr, (const uint8_t*)points + first * stride, n * stride);
                uint32_t blocks = (uint32_t)std::min<size_t>((n + 255) / 256, (size_t)gpu.sm_count() * 8);
                msm::pack_points_kernel<<<blocks, 256, 0, copy>>>(dr, stride, PB / 4, has_flag,
                                                                  d_points + b * slice_n * (PB / 4), (uint32_t)n);
                COUNT_LAUNCH();
                CUDA_OK(cudaGetLastError());
            }
            copied[b].record(copy);
            copied[b].wait(compute);
            if (unmont) unmont(ds, n, compute);
            m.slice(job, dp, ds, n, compute);
            consumed[b].record(compute);
        }
        m.finish(job, d_out, compute);
        compute.DtoH(out, d_out, JB);
        compute.sync();
        copy.sync();
        drain.armed = false;
    } catch (const cuda_error& e) {
        memset(out, 0, JB);                      // out->inf(), as the reference does on failure
        return rust_err(e.code(), e.what());
    } catch (const std::exception& e) {
        memset(out, 0, JB);
        return rust_err(-1, e.what());
    }
    return rust_ok();
}

// host points -> a plain cudaMalloc'ed buffer of packed affine rows that outlives the call
template<class F>
RustError msm_preload(const void* points, size_t npoints, size_t stride, bool has_flag, void** d_out)
{
    constexpr size_t PB = 2 * F::N * 4;
    *d_out = nullptr;
    try {
        const gpu_t& gpu = select_gpu(-1);
        gpu.select();
        if (stride < PB + (has_flag ? 1 : 0))
            return rust_err(-(int)cudaErrorInvalidValue, "msm: affine stride too small");
        if (stride % 4 != 0)
            return rust_err(-(int)cudaErrorInvalidValue, "msm: affine stride must be a multiple of 4 bytes");
        if (npoints >= (1ull << 31))
            return rust_err(-(int)cudaErrorInvalidValue, "msm: npoints must be < 2^31");
        const stream_t& copy = gpu[1];
        uint32_t* d_points = nullptr;
        CUDA_OK(cudaMalloc((void**)&d_points, npoints ? npoints * PB : 1));
        struct guard_t { uint32_t* p; ~guard_t() { if (p) (void)cudaFree(p); } } guard{d_points};
        const bool pageable = stager_t::is_pageable(points);
        std::unique_lock<std::mutex> stage_lock(gpu.stage_mtx, std::defer_lock);
        if (pageable) stage_lock.lock();
        auto upload = [&](void* dst, const void* src, size_t bytes) {
            if (pageable) gpu.stager().HtoD(copy, dst, src, bytes);
            else copy.HtoD(dst, src, bytes);
        };
        if (stride == PB && !has_flag) {
            upload(d_points, points, npoints * PB);
        } else {
            const size_t chunk = std::min<size_t>(npoints, (size_t)1 << 22);
            dev_ptr_t<uint8_t> d_raw(chunk * stride, copy);
            for (size_t first = 0; first < npoints; first += chunk) {
                const size_t n = std::min(chunk, npoints - first);
                upload(d_raw, (const uint8_t*)points + first * stride, n * stride);
                uint32_t blocks = (uint32_t)std::min<size_t>((n + 255) / 256, (size_t)gpu.sm_count() * 8);
                msm::pack_points_kernel<<<blocks, 256, 0, copy>>>(d_raw, stride, PB / 4, has_flag,
                                                                  d_points + first * (PB / 4), (uint32_t)n);
                COUNT_LAUNCH();
                CUDA_OK(cudaGetLastError());
            }
            copy.sync();
        }
        copy.sync();
        guard.p = nullptr;
        *d_out = d_points;
    } catch (const cuda_error& e) {
        return rust_err(e.code(), e.what());
    } catch (const std::exception& e) {
        return rust_err(-1, e.what());
    }
    return rust_ok();
}

template<class F>
RustError msm_dev(void* out, const void* d_points, size_t npoints, const void* d_scalars, void* stream)
{
    constexpr size_t JB = 3 * F::N * 4;
    try {
        const gpu_t& gpu = gpu_of_current_device();
        cudaStream_t s = (cudaStream_t)stream;
        const stream_t borrowed(s);
        dev_ptr_t<uint32_t> d_out(JB / 4, borrowed);           // released on every exit path
        msm::msm_t<F> m(gpu);
        m.invoke_dev(d_out, (const uint32_t*)d_points, npoints, (const uint32_t*)d_scalars, s);
        CUDA_OK(cudaMemcpyAsync(out, d_out, JB, cudaMemcpyDeviceToHost, s));
        CUDA_OK(cudaStreamSynchronize(s));
    } catch (const cuda_error& e) {
        memset(out, 0, JB);
        return rust_err(e.code(), e.what());
    } catch (const std::exception& e) {
        memset(out, 0, JB);
        return rust_err(-1, e.what());
    }
    return rust_ok();
}


// ---- synthetic inputs: out[i] = (i+1)*G, affine (role of util::generate_points_scalars,
// poc/msm-cuda/src/util.rs:11-38, which replicates 2^11 random points) ------------------------
template<class G>
__global__ void gen_points_kernel(uint32_t* out, uint32_t n)
{
    typedef typename G::F F;
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    ec::affine_t<F> g;
    for (int k = 0; k < F::N; k++) { g.X.l[k] = G::X(k); g.Y.l[k] = G::Y(k); }
    ec::xyzz_t<F> acc;
    acc.set_inf();
    for (int bit = 31 - __clz(i + 1); bit >= 0; bit--) {
        acc.dbl();
        if (((i + 1) >> bit) & 1) acc.madd(g);
    }
    F x = acc.X * acc.ZZ.inv(), y = acc.Y * acc.ZZZ.inv();
    for (int k = 0; k < F::N; k++) { out[(size_t)i * 2 * F::N + k] = x.l[k]; out[(size_t)i * 2 * F::N + F::N + k] = y.l[k]; }
}

template<class G>
RustError gen_points_dev(void* d_out, size_t n, void* stream)
{
    try {
        gen_points_kernel<G><<<(unsigned)((n + 63) / 64), 64, 0, (cudaStream_t)stream>>>((uint32_t*)d_out, (uint32_t)n);
        COUNT_LAUNCH();
        CUDA_OK(cudaGetLastError());
    } catch (const cuda_error& e) {
        return rust_err(e.code(), e.what());
    }
    return rust_ok();
}

// ---- sum of partial results (multi-GPU: every rank's Jacobian result -> one point) ----------
template<class F>
__global__ void combine_points_kernel(const uint32_t* partials, uint32_t count, uint32_t* out)
{
    if (blockIdx.x || threadIdx.x) return;
    ec::xyzz_t<F> acc;
    acc.set_inf();
    for (uint32_t i = 0; i < count; i++) {
        const uint32_t* p = partials + (size_t)i * 3 * F::N;
        ec::xyzz_t<F> q;
        F z;
        for (int k = 0; k < F::N; k++) { q.X.l[k] = p[k]; q.Y.l[k] = p[F::N + k]; z.l[k] = p[2 * F::N + k]; }
        q.ZZ = z.sqr();                      // Jacobian (X, Y, Z) == XYZZ (X, Y, Z^3, Z^2)
        q.ZZZ = q.ZZ * z;
        acc.add(q);
    }
    ec::jacobian_t<F> j = acc.to_jacobian();
    for (int k = 0; k < F::N; k++) { out[k] = j.X.l[k]; out[F::N + k] = j.Y.l[k]; out[2 * F::N + k] = j.Z.l[k]; }
}

template<class F>
RustError combine_host(void* out, const void* partials, size_t count)
{
    constexpr size_t JB = 3 * F::N * 4;
    try {
        const gpu_t& gpu = select_gpu(-1);
        const stream_t& s = gpu[0];
        dev_ptr_t<uint32_t> d_in(count * JB / 4, s), d_out(JB / 4, s);
        s.HtoD(d_in, partials, count * JB);
        combine_points_kernel<F><<<1, 32, 0, s>>>(d_in, (uint32_t)count, d_out);
        COUNT_LAUNCH();
        CUDA_OK(cudaGetLastError());
        s.DtoH(out, d_out, JB);
        s.sync();
    } catch (const cuda_error& e) {
        return rust_err(e.code(), e.what());
    }
    return rust_ok();
}

}  // namespace
