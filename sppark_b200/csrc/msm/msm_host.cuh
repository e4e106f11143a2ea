// MSM entry templates and the dispatch row each curve file builds from them (curve_row,
// curve_ops.cuh).  They take arguments msm.cu has checked, and throw what only the device can tell;
// the entry's guard turns that into its RustError.
// Host-pointer calls follow the reference's contract (msm/pippenger.cuh:730-747): scratch is
// allocated per call from the stream-ordered pool, scalars are 256-bit little-endian integers
// NOT in Montgomery form (mont=false), the result is a Jacobian point in Montgomery form.
#pragma once
#include "../ff/fields.cuh"
#include "curve_ops.cuh"
#include "msm.cuh"

namespace {

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

// The host <-> device copies of one call, on stream s.  A copy goes through the device's pinned
// stager iff its host side is pageable; a call with a pageable array among `host` holds the
// device's stage_mtx (one staged call at a time) for as long as it lives.
class host_copy_t {
    std::unique_lock<std::mutex> lock;
public:
    const gpu_t& gpu;
    const stream_t& s;
    host_copy_t(const gpu_t& gpu, const stream_t& s, std::initializer_list<const void*> host)
        : lock(gpu.stage_mtx, std::defer_lock), gpu(gpu), s(s)
    {
        for (const void* p : host)
            if (p != nullptr && stager_t::is_pageable(p)) { lock.lock(); break; }
    }
    void HtoD(void* dst, const void* src, size_t bytes) const
    {
        if (lock.owns_lock() && stager_t::is_pageable(src)) gpu.stager().HtoD(s, dst, src, bytes);
        else s.HtoD(dst, src, bytes);
    }
    void DtoH(void* dst, const void* src, size_t bytes) const
    {
        if (lock.owns_lock() && stager_t::is_pageable(dst)) gpu.stager().DtoH(s, dst, src, bytes);
        else s.DtoH(dst, src, bytes);
    }
};

// host rows [first, first + n) -> n packed {X, Y} rows at d_rows, on up's stream: one copy when
// the rows are packed already, else a copy to d_raw (n * stride bytes) that pack_points_kernel packs
template<class F>
void upload_rows(const host_copy_t& up, uint32_t* d_rows, uint8_t* d_raw, const host_rows& rows, size_t first,
                 size_t n)
{
    constexpr size_t PB = 2 * F::N * 4;
    const uint8_t* src = (const uint8_t*)rows.p + first * rows.stride;
    if (rows.stride == PB && !rows.has_flag) {
        up.HtoD(d_rows, src, n * PB);
        return;
    }
    up.HtoD(d_raw, src, n * rows.stride);
    const uint32_t blocks = (uint32_t)std::min<size_t>((n + 255) / 256, (size_t)up.gpu.sm_count() * 8);
    msm::pack_points_kernel<<<blocks, 256, 0, up.s>>>(d_raw, rows.stride, PB / 4, rows.has_flag, d_rows, (uint32_t)n);
    COUNT_LAUNCH();
    CUDA_OK(cudaGetLastError());
}

// The slices of a host-scalar MSM: a short first slice (the GPU idles while slice 0 crosses PCIe),
// then doubling ones (fewer bucket reloads); slice k+1 is copied while slice k is computed.
// `resident`: only the scalars cross PCIe.
inline std::vector<size_t> slice_schedule(size_t npoints, bool resident)
{
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
    return sched;
}

// MSM of host scalars.  The input is cut into slices (slice_schedule): slice k+1 is copied (copy
// stream, double-buffered) while slice k is sorted and folded into the persistent buckets (compute
// stream).  The reference overlaps the same way with its batches (msm/pippenger.cuh:505-557); here
// the bucket file is shared by all slices, so the running sums and the Horner pass run once at the
// end instead of once per batch.
// pts.d_rows set: the points are a context's device rows (msm_preload below -- the reference's
// msm_t{points, npoints} constructor + invoke(out, scalars), msm/pippenger.cuh:377-390,582-601), and
// only the scalars cross PCIe; with pts.copies > 1 they are a precomputed table, and slice k's points
// start at row `first` of every copy.
// scalar_bytes / nbits: the scalar format (msm_core.cuh Config); each slice uploads n * scalar_bytes.
// batch: vectors of npoints scalars one after the other, out one Jacobian point per vector.  They run
// in groups of msm_t::group_size vectors (Config::nvecs), each group sliced as one vector is: slice k
// of group q uploads its G rows of scalars on the copy stream while the unit before it computes.
template<class F, class Fr>
void msm_slices(void* out, const msm_points& pts, size_t npoints, const void* scalars, size_t batch, bool mont,
                uint32_t scalar_bytes, uint32_t nbits)
{
    constexpr size_t PB = 2 * F::N * 4, JB = 3 * F::N * 4;
    const gpu_t& gpu = select_gpu(-1);
    gpu.select();
    if (npoints == 0) { memset(out, 0, batch * JB); return; }
    const stream_t &compute = gpu[0], &copy = gpu[1];
    const uint32_t* resident = (const uint32_t*)pts.d_rows;
    const host_rows& rows = pts.host;
    const bool packed = resident || (rows.stride == PB && !rows.has_flag);

    const std::vector<size_t> sched = slice_schedule(npoints, resident != nullptr);
    const size_t nslices = sched.size();
    const size_t slice_n = *std::max_element(sched.begin(), sched.end());
    const msm::Config cfg1 = resident && pts.copies > 1
                                 ? msm::config_for_table(npoints, pts.wbits, pts.copies, pts.copy_stride, nbits,
                                                         scalar_bytes)
                                 : msm::make_config(npoints, nbits, scalar_bytes);
    const size_t G = msm::msm_t<F>::group_size(cfg1, slice_n, batch);
    const size_t nunits = (batch + G - 1) / G * nslices, nbuf = nunits > 1 ? 2 : 1;
    const host_copy_t up(gpu, copy, {rows.p, scalars});

    dev_ptr_t<uint32_t> d_out(batch * JB / 4, compute);
    const size_t SW = scalar_bytes / 4;                        // 32-bit words per scalar
    dev_ptr_t<uint32_t> d_points(resident ? 1 : nbuf * slice_n * (PB / 4), compute), d_scalars(nbuf * G * slice_n * SW, compute);
    dev_ptr_t<uint8_t> d_raw(packed ? 1 : nbuf * slice_n * rows.stride, compute);
    event_t copied[2], consumed[2], ready;
    ready.record(compute);                                    // buffers exist
    ready.wait(copy);
    drain_t drain(compute, copy);

    msm::msm_t<F> m(gpu);
    for (size_t v0 = 0, u = 0; v0 < batch; v0 += G) {
        const uint32_t g = (uint32_t)std::min(G, batch - v0);
        auto job = m.begin(msm::group_config(cfg1, g), slice_n, compute);
        size_t first = 0;
        for (size_t k = 0; k < nslices; first += sched[k], k++, u++) {
            const size_t b = u & (nbuf - 1), n = sched[k];
            const uint32_t* dp = resident ? resident + first * (PB / 4) : d_points + b * slice_n * (PB / 4);
            uint32_t* ds = d_scalars + b * G * slice_n * SW;
            if (u >= nbuf) consumed[b].wait(copy);                                // buffer free again
            // vector v0 + r of the group: its n scalars from `first` on, as row r of the buffer
            const uint8_t* src = (const uint8_t*)scalars + (v0 * npoints + first) * scalar_bytes;
            if (n == npoints) up.HtoD(ds, src, g * n * scalar_bytes);
            else for (uint32_t r = 0; r < g; r++) up.HtoD(ds + r * n * SW, src + r * npoints * scalar_bytes, n * scalar_bytes);
            if (!resident)
                upload_rows<F>(up, d_points + b * slice_n * (PB / 4), d_raw + b * slice_n * rows.stride, rows, first, n);
            copied[b].record(copy);
            copied[b].wait(compute);
            if (mont) scalars_from_mont<Fr>(ds, g * n, compute);
            m.slice(job, dp, ds, n, compute);
            consumed[b].record(compute);
        }
        m.finish(job, d_out + v0 * (JB / 4), compute);
    }
    compute.DtoH(out, d_out, batch * JB);
    compute.sync();
    copy.sync();
    drain.armed = false;
}

// host rows -> a plain cudaMalloc'ed buffer of packed affine rows that outlives the call, *d_out.
// *copies > 1: the buffer becomes the precomputed table of make_config_precomputed(npoints, *copies)
// (msm_table.cuh, copy-major rows); *copies and *wbits return the copy count stored and the width
// the table was built for.
template<class F>
void msm_preload(const host_rows& rows, size_t npoints, void** d_out, uint32_t* copies, uint32_t* wbits)
{
    constexpr size_t PB = 2 * F::N * 4;
    const gpu_t& gpu = select_gpu(-1);
    gpu.select();
    const msm::Config tcfg = *copies > 1 && npoints ? msm::make_config_precomputed(npoints, *copies)
                                                    : msm::make_config(npoints);
    const stream_t& copy = gpu[1];
    uint32_t* d_points = nullptr;
    CUDA_OK(cudaMalloc((void**)&d_points, npoints ? tcfg.copies * npoints * PB : 1));
    struct guard_t { uint32_t* p; ~guard_t() { if (p) (void)cudaFree(p); } } guard{d_points};
    const host_copy_t up(gpu, copy, {rows.p});
    const bool packed = rows.stride == PB && !rows.has_flag;
    {
        const size_t chunk = packed ? npoints : std::min<size_t>(npoints, (size_t)1 << 22);
        dev_ptr_t<uint8_t> d_raw(packed ? 1 : chunk * rows.stride, copy);
        for (size_t first = 0; first < npoints; first += chunk)
            upload_rows<F>(up, d_points + first * (PB / 4), d_raw, rows, first, std::min(chunk, npoints - first));
        if (!packed) copy.sync();
    }
    msm::build_table<F>(d_points, npoints, tcfg, copy);
    copy.sync();
    guard.p = nullptr;
    *d_out = d_points;
    *copies = tcfg.copies;
    *wbits = tcfg.wbits;
}

// batch: vectors of npoints device scalars one after the other (msm_t::invoke_dev), out one point per vector
template<class F>
void msm_dev(void* out, const void* d_points, size_t npoints, const void* d_scalars, size_t batch, void* stream,
             uint32_t scalar_bytes, uint32_t nbits)
{
    constexpr size_t JB = 3 * F::N * 4;
    const gpu_t& gpu = gpu_of_current_device();
    cudaStream_t s = (cudaStream_t)stream;
    const stream_t borrowed(s);
    dev_ptr_t<uint32_t> d_out(batch * JB / 4, borrowed);   // released on every exit path
    msm::msm_t<F> m(gpu);
    m.invoke_dev(d_out, (const uint32_t*)d_points, npoints, (const uint32_t*)d_scalars, s, nbits, scalar_bytes, batch);
    CUDA_OK(cudaMemcpyAsync(out, d_out, batch * JB, cudaMemcpyDeviceToHost, s));
    CUDA_OK(cudaStreamSynchronize(s));
}

// ---- scalar multiplication of point arrays (msm_scale.cuh) -------------------------------------
// device rows and scalars, enqueued on the caller's stream without a synchronisation
template<class F>
void scale_dev(void* d_out, const void* d_points, size_t npoints, const void* d_scalars, uint32_t scalar_bytes,
               uint32_t nbits, void* stream)
{
    (void)gpu_of_current_device();          // the device's pool and stack settings; fails without a device
    const stream_t s((cudaStream_t)stream);
    msm::scale_points<F>((uint32_t*)d_out, (const uint32_t*)d_points, npoints, (const uint32_t*)d_scalars,
                         scalar_bytes, nbits, s);
}

// host rows -> host packed rows.  Per chunk, on one stream: upload, the three steps in place on the
// uploaded rows, download.  The arithmetic outweighs the transfers many times over, so they are not
// overlapped.
template<class F>
void scale_host(void* out, const host_rows& rows, size_t npoints, const void* scalars, uint32_t scalar_bytes,
                uint32_t nbits)
{
    constexpr size_t PB = 2 * F::N * 4;
    const gpu_t& gpu = select_gpu(-1);
    gpu.select();
    const stream_t& s = gpu[0];
    const bool packed = rows.stride == PB && !rows.has_flag;
    const size_t chunk = std::min(npoints, msm::scale_chunk());
    dev_ptr_t<uint32_t> d_pts(chunk * (PB / 4), s), d_sc(chunk * scalar_bytes / 4, s);
    dev_ptr_t<uint8_t> d_raw(packed ? 1 : chunk * rows.stride, s);
    drain_t drain(s);
    const host_copy_t up(gpu, s, {rows.p, scalars, out});
    for (size_t first = 0; first < npoints; first += chunk) {
        const size_t n = std::min(chunk, npoints - first);
        up.HtoD(d_sc, (const uint8_t*)scalars + first * scalar_bytes, n * scalar_bytes);
        upload_rows<F>(up, d_pts, d_raw, rows, first, n);
        msm::scale_points<F>(d_pts, d_pts, n, d_sc, scalar_bytes, nbits, s);
        up.DtoH((uint8_t*)out + first * PB, d_pts, n * PB);
    }
    s.sync();
    drain.armed = false;
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
void gen_points(void* d_out, size_t n, void* stream)
{
    gen_points_kernel<G><<<(unsigned)((n + 63) / 64), 64, 0, (cudaStream_t)stream>>>((uint32_t*)d_out, (uint32_t)n);
    COUNT_LAUNCH();
    CUDA_OK(cudaGetLastError());
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
void combine(void* out, const void* partials, size_t count)
{
    constexpr size_t JB = 3 * F::N * 4;
    const gpu_t& gpu = select_gpu(-1);
    const stream_t& s = gpu[0];
    dev_ptr_t<uint32_t> d_in(count * JB / 4, s), d_out(JB / 4, s);
    s.HtoD(d_in, partials, count * JB);
    combine_points_kernel<F><<<1, 32, 0, s>>>(d_in, (uint32_t)count, d_out);
    COUNT_LAUNCH();
    CUDA_OK(cudaGetLastError());
    s.DtoH(out, d_out, JB);
    s.sync();
}

// the row of one curve: G its generator, whose F is the base field (an fp2_t for G2), Fr its scalar field
template<class G, class Fr>
constexpr curve_ops curve_row()
{
    typedef typename G::F F;
    return {msm_slices<F, Fr>, msm_dev<F>, msm_preload<F>, scale_host<F>, scale_dev<F>, gen_points<G>, combine<F>,
            2 * F::N * 4, 3 * F::N * 4};
}

}  // namespace
