/*
 * oracle/ref_msm_cpu.cpp -- TEST INFRASTRUCTURE ONLY.
 *
 * Thin extern "C" door onto the REFERENCE's own CPU Pippenger, compiled from
 * the sources where they lie in the reference tree (msm/pippenger.hpp:218,
 * ec/*.hpp, util/thread_pool_t.hpp) with oracle/shim/blst_t.hpp supplying the
 * un-vendored blst host field.  Built into oracle/_ref/ by oracle/Makefile;
 * used to validate the C restatement (oracle/msm.c) and as the "reference"
 * CPU baseline of bench.py.
 */
#include <blst_t.hpp>
#include <ff/bls12-381.hpp>
#include <ec/jacobian_t.hpp>
#include <ec/xyzz_t.hpp>

typedef jacobian_t<fp_t> point_t;
typedef xyzz_t<fp_t> bucket_t;
typedef bucket_t::affine_t affine_t;
typedef fr_t scalar_t;

#include <msm/pippenger.hpp>

static thread_pool_t* pool_of(int nthreads)
{
    static thread_pool_t* pool = nullptr;
    static int cur = -1;
    if (nthreads < 2)
        return nullptr;
    if (pool == nullptr || cur != nthreads) {
        delete pool;
        pool = new thread_pool_t((unsigned)nthreads);
        cur = nthreads;
    }
    return pool;
}

extern "C" int ref_cpu_threads()
{
    thread_pool_t p;
    return (int)p.size();
}

/* points: 96-byte {X,Y} Montgomery; scalars: 32-byte LE, not Montgomery;
 * out: 144-byte {X,Y,Z} */
extern "C" void ref_cpu_mult_pippenger(void* out, const void* points, size_t npoints,
                                       const void* scalars, int nthreads)
{
    point_t ret;
    mult_pippenger<bucket_t>(ret, (const affine_t*)points, npoints,
                             (const scalar_t*)scalars, false, pool_of(nthreads));
    memcpy(out, &ret, sizeof(ret));
}

extern "C" void ref_cpu_naive(void* out, const void* points, size_t npoints, const void* scalars)
{
    point_t acc, t;
    acc.inf();
    for (size_t i = 0; i < npoints; i++) {
        mult(t, ((const affine_t*)points)[i],
             reinterpret_cast<const unsigned char*>(&((const scalar_t*)scalars)[i]), 255);
        acc.add(t);
    }
    memcpy(out, &acc, sizeof(acc));
}
