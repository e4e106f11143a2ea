/*
 * oracle/ref_poly.cu -- TEST INFRASTRUCTURE ONLY.
 * Host-pointer doors onto the REFERENCE's own polynomial helpers, compiled from the reference
 * sources where they lie (polynomial/prefix_op.cuh:322, polynomial/div_by_x_minus_z.cuh:445,
 * polynomial/evaluate.cuh:308).  The reference ships no test or golden vector for these
 * templates, so tests/golden/make_golden.py runs them on a GPU through this shim and commits
 * the input/output pairs (tests/golden/poly_ref_gpu.npz) -- that is what pins oracle/poly.py.
 */
#if defined(FEATURE_GOLDILOCKS)
# include <ff/goldilocks.hpp>
#elif defined(FEATURE_BABY_BEAR)
# include <ff/baby_bear.hpp>
#elif defined(FEATURE_BLS12_381)
# include <ff/bls12-381.hpp>
#endif
#include <util/gpu_t.cuh>
#include <polynomial/prefix_op.cuh>
#include <polynomial/div_by_x_minus_z.cuh>
#include <polynomial/evaluate.cuh>

extern "C" int ref_poly_elem_bytes() { return (int)sizeof(fr_t); }

/* op: 0 = Add, 1 = Multiply; inclusive prefix, in place on a host buffer */
extern "C" int ref_prefix_op(int op, void* inout, size_t len)
{
    try {
        auto& gpu = select_gpu(0);
        dev_ptr_t<fr_t> d{len, gpu[0]};
        gpu[0].HtoD(&d[0], (const fr_t*)inout, len);
        if (op == 0) prefix_op<Add<fr_t>>(&d[0], (const fr_t*)&d[0], len, gpu[0]);
        else         prefix_op<Multiply<fr_t>>(&d[0], (const fr_t*)&d[0], len, gpu[0]);
        gpu[0].DtoH((fr_t*)inout, &d[0], len);
        gpu[0].sync();
        return 0;
    } catch (const cuda_error& e) {
        return e.code();
    }
}

extern "C" int ref_div_by_x_minus_z(void* inout, size_t len, const void* z, int rotate)
{
    try {
        auto& gpu = select_gpu(0);
        dev_ptr_t<fr_t> d{len, gpu[0]};
        gpu[0].HtoD(&d[0], (const fr_t*)inout, len);
        if (rotate) div_by_x_minus_z<true>(&d[0], len, *(const fr_t*)z, gpu[0]);
        else        div_by_x_minus_z<false>(&d[0], len, *(const fr_t*)z, gpu[0]);
        gpu[0].DtoH((fr_t*)inout, &d[0], len);
        gpu[0].sync();
        return 0;
    } catch (const cuda_error& e) {
        return e.code();
    }
}

extern "C" int ref_evaluate(void* ret, const void* x, size_t n, const void* coeffs, size_t len)
{
    try {
        auto& gpu = select_gpu(0);
        dev_ptr_t<fr_t> d_c{len, gpu[0]}, d_x{n, gpu[0]}, d_r{n, gpu[0]};
        gpu[0].HtoD(&d_c[0], (const fr_t*)coeffs, len);
        gpu[0].HtoD(&d_x[0], (const fr_t*)x, n);
        evaluate(&d_r[0], (const fr_t*)&d_x[0], n, (const fr_t*)&d_c[0], len, gpu[0]);
        gpu[0].DtoH((fr_t*)ret, &d_r[0], n);
        gpu[0].sync();
        return 0;
    } catch (const cuda_error& e) {
        return e.code();
    }
}

/* device-pointer forms, enqueued on the reference's stream and synchronised by the caller through
 * ref_poly_sync(): tools/probe_poly.py times the reference's kernels with data resident in HBM */
extern "C" void* ref_poly_stream() { return (void*)(cudaStream_t)select_gpu(0)[0]; }
extern "C" int ref_poly_sync()
{
    try { select_gpu(0)[0].sync(); return 0; } catch (const cuda_error& e) { return e.code(); }
}
extern "C" int ref_prefix_op_dev(int op, void* d_inout, size_t len)
{
    try {
        auto& gpu = select_gpu(0);
        if (op == 0) prefix_op<Add<fr_t>>((fr_t*)d_inout, (const fr_t*)d_inout, len, gpu[0]);
        else         prefix_op<Multiply<fr_t>>((fr_t*)d_inout, (const fr_t*)d_inout, len, gpu[0]);
        return 0;
    } catch (const cuda_error& e) {
        return e.code();
    }
}
extern "C" int ref_div_by_x_minus_z_dev(void* d_inout, size_t len, const void* z, int rotate)
{
    try {
        auto& gpu = select_gpu(0);
        if (rotate) div_by_x_minus_z<true>((fr_t*)d_inout, len, *(const fr_t*)z, gpu[0]);
        else        div_by_x_minus_z<false>((fr_t*)d_inout, len, *(const fr_t*)z, gpu[0]);
        return 0;
    } catch (const cuda_error& e) {
        return e.code();
    }
}
extern "C" int ref_evaluate_dev(void* d_ret, const void* d_x, size_t n, const void* d_coeffs, size_t len)
{
    try {
        auto& gpu = select_gpu(0);
        evaluate((fr_t*)d_ret, (const fr_t*)d_x, n, (const fr_t*)d_coeffs, len, gpu[0]);
        return 0;
    } catch (const cuda_error& e) {
        return e.code();
    }
}
