/*
 * oracle/ref_msm_g2.cu -- TEST INFRASTRUCTURE ONLY.
 *
 * Harness around the reference's OWN templates (msm/pippenger.cuh, ff/bls12-381-fp2.hpp, ec/ *.hpp,
 * included from where they lie under $(REF)) instantiating the G2 MSM on PACKED affine points
 * (xyzz_t<fp2_t>::affine_t, 192 bytes, infinity = X == Y == 0).
 *
 * Why not the reference's mult_pippenger_fp2_inf itself (poc/msm-cuda/cuda/pippenger_inf.cu:41-47,
 * built as _ref/libref_msm_g2_gpu.so)?  Its Affine_inf_t<fp2_t>::mem_t (ec/affine_t.hpp:95-97) is
 * sized from sizeof(field_t), which is 96 bytes in nvcc's host pass (host fp2_t = vec384x) but 48
 * in the device pass (device fp2_t = one fp_mont per lane): the host copies points with a
 * 224-byte pitch, the kernels index them with 208.  Recorded on a GPU (tests/golden/
 * make_golden.py g2): n = 1 is right, n = 2 returns s0*P0, n >= 33 is not even on the curve.
 * The packed affine_t has no such field, so this instantiation is consistent and pins G2.
 */
#include <cuda.h>
#if defined(FEATURE_BN254)               /* the msm crate's other two features: same harness, their Fp2 */
# include <ff/alt_bn128-fp2.hpp>
#elif defined(FEATURE_BLS12_377)
# include <ff/bls12-377-fp2.hpp>
#else
# include <ff/bls12-381-fp2.hpp>
#endif
#include <ec/jacobian_t.hpp>
#include <ec/xyzz_t.hpp>

/* msm/pippenger.cuh explicitly instantiates its G1 kernels for these four global names */
using bucket_t = xyzz_t<fp_t>;
using point_t = jacobian_t<fp_t>;
using affine_t = bucket_t::affine_t;
using scalar_t = fr_t;

#include <msm/pippenger.cuh>

using g2_bucket_t = xyzz_t<fp2_t>;
using g2_point_t = jacobian_t<fp2_t>;
using g2_affine_t = g2_bucket_t::affine_t;    /* packed: x, y in Fp2, infinity = all zero */

/* not guarded by __CUDA_ARCH__: the device pass must see the call to instantiate the fp2 kernels
 * (the reference's explicit instantiations, msm/pippenger.cuh:299-316, cover bucket_t only) */
extern "C" RustError::by_value ref_mult_pippenger_fp2(g2_point_t* sum, const g2_affine_t* rows, size_t n,
                                                      const scalar_t* k)
{
    const bool scalars_in_montgomery_form = false;
    RustError status = mult_pippenger<g2_bucket_t>(sum, rows, n, k, scalars_in_montgomery_form);
    return status;
}
