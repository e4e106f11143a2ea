// BLS12-381 G1 MSM (its drop-in entry points of poc/msm-cuda are in msm.cu) and the device self-test hooks.
#include "msm_host.cuh"

constexpr curve_ops curve_bls12_381 = curve_row<ff::bls12_381_g1_gen, ff::bls12_381_fr_t>();

// ---- device self-test hook: element-wise field ops through the PTX arithmetic -------------
// op 0 mul, 1 add, 2 sub, 3 sqr, 4 mul_shared, 5 sqr_shared, 6 msub_shared(x,y,y,x^2): host arrays
// of n elements.  op 7 msub_shared with four independent operands: a = (a_i, c_i) and b = (b_i, d_i)
// interleaved, 2n elements each, r_i = a_i*b_i - c_i*d_i.  Used by the GPU KAT tests.
template<class F>
__global__ void selftest_kernel(int op, size_t n, uint32_t* r, const uint32_t* a, const uint32_t* b)
{
    size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    F x, y, z;
    if (op == 7) {
        F c, d;
        for (int k = 0; k < F::N; k++) {
            x.l[k] = a[2 * i * F::N + k]; c.l[k] = a[(2 * i + 1) * F::N + k];
            y.l[k] = b[2 * i * F::N + k]; d.l[k] = b[(2 * i + 1) * F::N + k];
        }
        z = F::msub_shared(x, y, c, d);
        for (int k = 0; k < F::N; k++) r[i * F::N + k] = z.l[k];
        return;
    }
    for (int k = 0; k < F::N; k++) { x.l[k] = a[i * F::N + k]; y.l[k] = b[i * F::N + k]; }
    switch (op) {
    case 0: z = x * y; break;
    case 1: z = x + y; break;
    case 2: z = x - y; break;
    case 3: z = x.sqr(); break;
    case 4: z = F::mul_shared(x, y); break;            // Karatsuba wide product + separate reduction
    case 5: z = F::sqr_shared(x); break;               // dedicated squaring
    default: z = F::msub_shared(x, y, y, x.sqr()); break;   // x*y - y*x^2, one reduction
    }
    for (int k = 0; k < F::N; k++) r[i * F::N + k] = z.l[k];
}

template<class F>
static void selftest(int op, size_t n, void* r, const void* a, const void* b)
{
    const gpu_t& gpu = select_gpu(-1);
    const stream_t& s = gpu[0];
    const size_t bytes = n * F::N * 4, in_bytes = op == 7 ? 2 * bytes : bytes;
    dev_ptr_t<uint32_t> da(in_bytes / 4, s), db(in_bytes / 4, s), dr(n * F::N, s);
    s.HtoD(da, a, in_bytes);
    s.HtoD(db, b, in_bytes);
    selftest_kernel<F><<<(unsigned)((n + 127) / 128), 128, 0, s>>>(op, n, dr, da, db);
    COUNT_LAUNCH();
    CUDA_OK(cudaGetLastError());
    s.DtoH(r, dr, bytes);
    s.sync();
}

extern "C" RustError sppark_b200_selftest_field(int field, int op, size_t n, void* r, const void* a, const void* b)
{
    return guarded([&] {
        switch (field) {
        case 0: selftest<ff::bls12_381_fp_t>(op, n, r, a, b); break;
        case 1: selftest<ff::bls12_381_fr_t>(op, n, r, a, b); break;
        case 2: selftest<ff::pallas_fp_t>(op, n, r, a, b); break;
        case 3: selftest<ff::vesta_fp_t>(op, n, r, a, b); break;
        case 4: selftest<ff::bn254_fp_t>(op, n, r, a, b); break;
        case 5: selftest<ff::bn254_fr_t>(op, n, r, a, b); break;
        case 6: selftest<ff::bls12_377_fp_t>(op, n, r, a, b); break;
        case 7: selftest<ff::bls12_377_fr_t>(op, n, r, a, b); break;
        default: throw cuda_error(-(int)cudaErrorInvalidValue, "selftest: unknown field");
        }
        return rust_ok();
    });
}

// ---- device self-test hook: the MSM's bucket sort alone (tests/test_msm_sort.py) -------------------
// Host scalars (n x 8 words); window width wbits, heavy threshold as make_config(n); cap entries per
// bin-sort CTA (0 = the default).  Host outputs: counts / offsets (nwins << (wbits-1)), sorted
// (nwins * n), heavy_slots (one slot per heavy bucket), info = {nwins, heavy threshold, #heavy,
// lg_bins, #overflow bins}.
extern "C" RustError sppark_b200_selftest_msm_sort(size_t n, uint32_t wbits, uint32_t cap, const void* scalars,
                                                   void* counts, void* offsets, void* sorted, void* heavy_slots,
                                                   uint32_t* info)
{
    using namespace msm;
    return guarded([&] {
        if (n == 0 || n >= (1ull << 31) || wbits < 3 || wbits > 24 || cap > SORT_CAP)
            throw cuda_error(-(int)cudaErrorInvalidValue, "selftest_msm_sort: bad arguments");
        const gpu_t& gpu = select_gpu(-1);
        const stream_t& s = gpu[0];
        Config cfg = make_config(n);
        cfg.wbits = wbits;
        cfg.nwins = (256 + wbits - 1) / wbits;
        cfg.lg_nb = wbits - 1;
        const size_t nslots = (size_t)cfg.nwins << cfg.lg_nb, entries = (size_t)cfg.nwins * n;
        const size_t nbins = (size_t)cfg.nwins << sort_lg_bins(cfg, n);
        const size_t heavy_cap = entries / (cfg.heavy + 1) + 1, chunk_cap = entries / cfg.heavy_chunk + heavy_cap;
        dev_ptr_t<uint32_t> d_sc(8 * n, s), d_counts(nslots, s), d_offsets(nslots, s), d_cursor(nslots, s);
        dev_ptr_t<uint32_t> d_ctrl(4, s), d_heavy(3 * heavy_cap, s), d_cmap(chunk_cap, s), d_sorted(entries, s);
        dev_ptr_t<uint32_t> d_bcount(nbins, s), d_bbase(nbins, s), d_bcur(nbins, s), d_over(nbins, s);
        dev_ptr_t<uint32_t> d_staging(2 * entries, s);
        s.HtoD(d_sc, scalars, 32 * n);
        const SortBufs sb{d_counts, d_offsets, d_cursor, d_ctrl, d_heavy, d_cmap, d_sorted,
                          d_bcount, d_bbase, d_bcur, d_over, reinterpret_cast<uint2*>((uint32_t*)d_staging)};
        sort_slice(cfg, cap ? cap : SORT_CAP, d_sc, sb, (uint32_t)gpu.sm_count(), s);
        uint32_t ctrl[4];
        s.DtoH(ctrl, d_ctrl, 16);
        s.DtoH(counts, d_counts, nslots * 4);
        s.DtoH(offsets, d_offsets, nslots * 4);
        s.DtoH(sorted, d_sorted, entries * 4);
        s.sync();
        std::vector<uint32_t> hl(3 * (size_t)ctrl[1] + 1);
        if (ctrl[1]) s.DtoH(hl.data(), d_heavy, 12 * (size_t)ctrl[1]);
        s.sync();
        for (uint32_t h = 0; h < ctrl[1]; h++) static_cast<uint32_t*>(heavy_slots)[h] = hl[3 * h];
        info[0] = cfg.nwins; info[1] = cfg.heavy; info[2] = ctrl[1]; info[3] = sort_lg_bins(cfg, n); info[4] = ctrl[3];
        return rust_ok();
    });
}
