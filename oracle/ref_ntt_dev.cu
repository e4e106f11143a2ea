/*
 * oracle/ref_ntt_dev.cu -- TEST INFRASTRUCTURE ONLY.
 * Device-pointer door onto the REFERENCE's own NTT (ntt/ntt.cuh:344-350 Base_dev_ptr),
 * compiled from the reference sources where they lie.  Lets bench/probe scripts time the
 * reference's kernels on the same GPU with data already resident ("the bar to beat").
 */
#if defined(FEATURE_GOLDILOCKS)
# include <ff/goldilocks.hpp>
#elif defined(FEATURE_BABY_BEAR)
# include <ff/baby_bear.hpp>
#elif defined(FEATURE_BLS12_381)
# include <ff/bls12-381.hpp>
#endif
#include <ntt/ntt.cuh>

extern "C" int ref_ntt_dev(void* d_inout, uint32_t lg, int order, int direction, int type)
{
    try {
        auto& gpu = select_gpu(0);
        NTT::Base_dev_ptr(gpu[0], (fr_t*)d_inout, lg, (NTT::InputOutputOrder)order,
                          (NTT::Direction)direction, (NTT::Type)type);
        gpu[0].sync();
        return 0;
    } catch (const cuda_error& e) {
        return e.code();
    }
}
/* enqueue only (no sync), for event timing by the caller on the same stream */
extern "C" void* ref_ntt_stream()
{   return (void*)(cudaStream_t)select_gpu(0)[0];   }
extern "C" int ref_ntt_dev_async(void* d_inout, uint32_t lg, int order, int direction, int type)
{
    try {
        auto& gpu = select_gpu(0);
        NTT::Base_dev_ptr(gpu[0], (fr_t*)d_inout, lg, (NTT::InputOutputOrder)order,
                          (NTT::Direction)direction, (NTT::Type)type);
        return 0;
    } catch (const cuda_error& e) {
        return e.code();
    }
}

/* the reference's own low-degree extension (ntt/ntt.cuh:336-338), host buffer of 2^(lg+lb) elements */
extern "C" int ref_lde(void* inout, uint32_t lg, uint32_t lg_blowup)
{
    RustError e = NTT::LDE(select_gpu(0), (fr_t*)inout, lg, lg_blowup);
    if (e.message) free(e.message);
    return e.code;
}
