/*
 * sppark_b200.h -- C ABI of libsppark_b200.so, the H100-native (sm_90a) MSM / NTT library.
 *
 * The first block is the DROP-IN surface: the exact symbols, signatures and error
 * convention that supranational/sppark's PoC crates bind through FFI, so that a caller of
 * the reference links against this library unchanged.  Each declaration cites the
 * reference interface it replaces (paths relative to the sppark tree).
 *
 * The second block (sppark_b200_*) is this library's extended surface: the same operations
 * on DEVICE pointers and an explicit CUDA stream (the reference reaches these through C++
 * only: NTT::Base_dev_ptr ntt/ntt.cuh:344-350, msm_t::invoke with device pointers
 * msm/pippenger.cuh:582-601), other fields/curves, and introspection for tests.
 *
 * Conventions (util/rusterror.h:18-36, util/exception.cuh:12-21, rust/src/lib.rs:9-22):
 *   - every entry point returns RustError BY VALUE; code == 0 is success, otherwise
 *     -(cudaError_t) or a negative errno-style code; message is NULL or a malloc()ed C
 *     string owned by the caller (free() / drop_error_message()).
 *   - no C++ exception ever crosses this boundary.
 *   - all pointers are caller-owned; host pointers unless the name says _dev.
 *   - there is NO CPU fallback: without a usable CUDA device every call fails with
 *     code -cudaErrorNoDevice (-100).
 */
#ifndef SPPARK_B200_H
#define SPPARK_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct RustError {
    int   code;
    char *message;
#ifdef __cplusplus
    typedef struct RustError by_value;         /* the reference's RustError::by_value: same two words */
#endif
} RustError;                                   /* util/rusterror.h:18-36 */

/* --- memory layouts (ABI) ---------------------------------------------------------
 * fp  (BLS12-381 base field): 12 x uint32 little-endian limbs = 48 B, Montgomery form,
 *     R = 2^384   (ff/mont_t.cuh:36, ff/bls12-381.hpp:14-30)
 * fr  (scalars): 8 x uint32 LE limbs = 32 B, plain (non-Montgomery) integers < r
 * affine      {X, Y}                96 B, infinity = all-zero     (ec/affine_t.hpp:19-72)
 * affine_inf  {X, Y, bool inf}     host stride ffi_affine_sz (104 for arkworks G1Affine),
 *                                   inf = bit 0 of the byte at +96 (ec/affine_t.hpp:74-122)
 * jacobian    {X, Y, Z}            144 B, infinity = Z == 0       (ec/jacobian_t.hpp:16-58)
 * xyzz        {X, Y, ZZZ, ZZ}      192 B (internal buckets)       (ec/xyzz_t.hpp:16-17)
 * gl64        uint64 canonical (< p), not Montgomery              (ff/gl64_t.cuh:39-60)
 * bb31        uint32 Montgomery residue, R = 2^32                 (ff/mont32_t.cuh:20-41)
 */

enum { SPPARK_NTT_NN = 0, SPPARK_NTT_NR = 1, SPPARK_NTT_RN = 2, SPPARK_NTT_RR = 3,
                                               /* NTT::InputOutputOrder, ntt/ntt.cuh:33.  RR follows
                                                  the reference: same transform as NN (its tests
                                                  assert NN == RR), bit-reversed coset exponents */
       SPPARK_NTT_BB = 4 };                    /* extension: bit-reversed input AND output */
enum { SPPARK_NTT_FORWARD = 0, SPPARK_NTT_INVERSE = 1 };   /* NTT::Direction, ntt/ntt.cuh:34 */
enum { SPPARK_NTT_STANDARD = 0, SPPARK_NTT_COSET = 1 };    /* NTT::Type,      ntt/ntt.cuh:35 */

/* ================================ drop-in surface ================================= */

/* (C++ callers that DEFINE these entry points themselves, with their own typed signatures, on
 * top of include/sppark_b200.hpp -- the reference's poc glue does -- hide the four declarations
 * below with SPPARK_B200_NO_DROPIN_DECLS.) */
#ifndef SPPARK_B200_NO_DROPIN_DECLS
/* poc/msm-cuda/cuda/pippenger.cu:20-25 ; Rust decl poc/msm-cuda/src/lib.rs:24-29.
 * BLS12-381 G1: out = sum scalars[i] * points[i]. */
RustError mult_pippenger(void *out_jacobian, const void *points_affine, size_t npoints,
                         const void *scalars);

/* poc/msm-cuda/cuda/pippenger_inf.cu:28-34 ; Rust decl poc/msm-cuda/src/lib.rs:52-58.
 * Same, points carry an explicit infinity flag and a host stride. */
RustError mult_pippenger_inf(void *out_jacobian, const void *points_affine_inf, size_t npoints,
                             const void *scalars, size_t ffi_affine_sz);

/* poc/msm-cuda/cuda/pippenger_inf.cu:36-47 ; Rust decl poc/msm-cuda/src/lib.rs:84-119.
 * BLS12-381 G2 (coordinates in Fp2 = two consecutive Fp, blst_fp2 / arkworks Fq2 layout):
 * out is a 288-byte Jacobian point, points are arkworks G2Affine (x, y, infinity flag) with a
 * host stride of ffi_affine_sz bytes. */
RustError mult_pippenger_fp2_inf(void *out_jacobian, const void *points_affine_inf, size_t npoints,
                                 const void *scalars, size_t ffi_affine_sz);

/* poc/ntt-cuda/cuda/ntt_api.cu:25-36 (FEATURE_GOLDILOCKS build, the one
 * poc/ntt-cuda/go/goldilocks.go:24-40 loads); in place on HOST memory; lg == 0 is a no-op. */
RustError compute_ntt(size_t device_id, void *inout, uint32_t lg_domain_size,
                      int ntt_order, int ntt_direction, int ntt_type);
#endif /* SPPARK_B200_NO_DROPIN_DECLS */

/* util/all_gpus.cpp:65-86 */
int  cuda_available(void);                     /* bool in the reference */
void drop_error_message(char *msg);

/* util/all_gpus.cpp:69-79 -- reference-counted device allocations crossing the FFI (Rust
 * `Gpu_Ptr<T>`, rust/src/lib.rs:62-97).  A handle is one pointer-sized word. */
typedef struct { void *inner; } gpu_ptr_t;
void      drop_gpu_ptr_t(gpu_ptr_t *by_ref);
gpu_ptr_t clone_gpu_ptr_t(const gpu_ptr_t *by_ref);

/* ================================ extended surface ================================ */

/* companions of gpu_ptr_t (the reference creates these from C++ only) */
gpu_ptr_t sppark_b200_gpu_ptr_alloc(size_t bytes);           /* {NULL} on failure */
void     *sppark_b200_gpu_ptr_get(const gpu_ptr_t *by_ref);  /* the device pointer */
size_t    sppark_b200_gpu_ptr_refs(const gpu_ptr_t *by_ref);

enum { SPPARK_FIELD_GL64 = 0, SPPARK_FIELD_BB31 = 1,
       /* 256-bit Montgomery scalar fields, 8 x uint32 limbs per element (the reference's "wide"
        * NTT kernels, ntt/kernels/{ct,gs}_mixed_radix_wide.cu): fr of FEATURE_BLS12_381,
        * FEATURE_PALLAS (= Vesta's base field) and FEATURE_VESTA (= Pallas' base field) */
       SPPARK_FIELD_BLS12_381_FR = 2, SPPARK_FIELD_PALLAS_FR = 3, SPPARK_FIELD_VESTA_FR = 4,
       /* FEATURE_BN254 (ff/alt_bn128.hpp, domains up to 2^28), FEATURE_BLS12_377 (ff/bls12-377.hpp) */
       SPPARK_FIELD_BN254_FR = 5, SPPARK_FIELD_BLS12_377_FR = 6 };
enum { SPPARK_CURVE_BLS12_381_G1 = 0, SPPARK_CURVE_PALLAS = 1, SPPARK_CURVE_VESTA = 2,
       SPPARK_CURVE_BLS12_381_G2 = 3,
       /* the other two G1 groups poc/msm-cuda builds (features bn254, bls12_377; Cargo.toml:12-17) */
       SPPARK_CURVE_BN254_G1 = 4, SPPARK_CURVE_BLS12_377_G1 = 5,
       /* and their G2 groups (mult_pippenger_fp2_inf of those builds, pippenger_inf.cu:8-13,36-47):
        * Fp2 = Fp[u]/(u^2 + 1) for BN254 (ff/alt_bn128-fp2.hpp), Fp[u]/(u^2 + 5) for BLS12-377
        * (ff/bls12-377-fp2.hpp); coordinates are (c0, c1) pairs of base-field Montgomery limbs */
       SPPARK_CURVE_BN254_G2 = 6, SPPARK_CURVE_BLS12_377_G2 = 7 };

/* compute_ntt for any single-word field (the reference builds one .so per FEATURE_*) */
RustError sppark_b200_ntt(int field, size_t device_id, void *inout, uint32_t lg_domain_size,
                          int ntt_order, int ntt_direction, int ntt_type);
/* NTT::Base_dev_ptr (ntt/ntt.cuh:344-350): d_inout is device memory, work is enqueued on
 * `stream` (a cudaStream_t; NULL = legacy default stream) and NOT synchronised. */
RustError sppark_b200_ntt_dev(int field, void *d_inout, uint32_t lg_domain_size,
                              int ntt_order, int ntt_direction, int ntt_type, void *stream);

/* Low-degree extension, NTT::LDE / NTT::LDE_aux (ntt/ntt.cuh:247-340; SURVEY.md section 8f row 1):
 * inout holds 2^lg evaluations and has room for 2^(lg + lg_blowup) elements; it returns the
 * evaluations of the same polynomial on the coset group_gen*<w_(2^(lg+lg_blowup))>, natural order.
 * aux_out (NULL or 2^lg elements) receives the coefficients in natural order. */
RustError sppark_b200_lde(int field, size_t device_id, void *inout, uint32_t lg_domain_size,
                          uint32_t lg_blowup, void *aux_out);

/* The device-pointer halves of the same step, NTT::LDE_powers / NTT::LDE_expand
 * (ntt/ntt.cuh:352-365), enqueued on `stream`, not synchronised:
 *   lde_powers: d_inout[i] *= group_gen^bitrev(i), i < 2^lg (coefficients in bit-reversed order);
 *   lde_expand: d_out[i << lg_blowup] = d_in[i], zero elsewhere (no coset shift); d_in may be the
 *               tail of d_out, as the reference allows. */
RustError sppark_b200_lde_powers_dev(int field, void *d_inout, uint32_t lg_domain_size, void *stream);
RustError sppark_b200_lde_expand_dev(int field, void *d_out, const void *d_in, uint32_t lg_domain_size,
                                     uint32_t lg_blowup, void *stream);

/* Batched NTT and LDE (the reference has no batched entry): `batch` transforms of 2^lg elements
 * each, stored one after another (row b = elements [b * 2^lg, (b + 1) * 2^lg)) in the field's memory
 * format.  Every row comes out exactly as the single-transform entry with the same order, direction
 * and type returns it.  lg == 0 or batch == 0 is a no-op; a byte size that overflows size_t is
 * rejected before any memory is touched.
 *   ntt_batch_dev: device memory, in place, enqueued on `stream`, not synchronised;
 *   lde_batch_dev: d_in = batch x 2^lg evaluations, overwritten with each row's coefficients in
 *                  bit-reversed order; d_out = batch x 2^(lg + lg_blowup) evaluations on the coset,
 *                  natural order (per row what sppark_b200_lde returns); the two must not overlap;
 *                  enqueued on `stream`;
 *   ntt_batch:     host memory, in place, synchronised; groups of rows are uploaded, transformed and
 *                  downloaded in a pipeline (pinned or registered memory overlaps copies and work). */
RustError sppark_b200_ntt_batch_dev(int field, void *d_inout, uint32_t lg_domain_size, size_t batch,
                                    int ntt_order, int ntt_direction, int ntt_type, void *stream);
RustError sppark_b200_lde_batch_dev(int field, void *d_out, void *d_in, uint32_t lg_domain_size,
                                    uint32_t lg_blowup, size_t batch, void *stream);
RustError sppark_b200_ntt_batch(int field, size_t device_id, void *inout, uint32_t lg_domain_size,
                                size_t batch, int ntt_order, int ntt_direction, int ntt_type);

/* NTT and LDE down the COLUMNS of a row-major matrix (Goldilocks and BabyBear only; the 256-bit
 * fields are refused with -cudaErrorInvalidValue): height = 2^lg_domain_size rows, `width` >= 1
 * columns, element (i, c) at word i * width + c, in the field's memory format.  Column c of the result
 * is exactly what the single-transform entry with the same order, direction and type returns for
 * column c alone; no transpose is made.  lg == 0 or width == 0 is a no-op; a byte size that overflows
 * size_t, an lg (or lg + lg_blowup) past the field's maximum, a bad order / direction / type, an
 * unknown field or overlapping LDE buffers are rejected before any memory is touched.
 *   ntt_matrix_dev: device memory, in place, enqueued on `stream`, not synchronised;
 *   lde_matrix_dev: d_in = 2^lg x width evaluations, left holding each column's coefficients in
 *                   bit-reversed row order (column c of d_in = row c of what lde_batch_dev leaves in
 *                   its d_in); d_out = 2^(lg + lg_blowup) x width evaluations on the coset, natural
 *                   order; no overlap with d_in; enqueued on `stream`;
 *   ntt_matrix:     host memory, in place, synchronised: the whole matrix is uploaded, transformed and
 *                   downloaded (pageable memory through the same staging as the other host entries). */
RustError sppark_b200_ntt_matrix_dev(int field, void *d_inout, uint32_t lg_domain_size, size_t width,
                                     int ntt_order, int ntt_direction, int ntt_type, void *stream);
RustError sppark_b200_lde_matrix_dev(int field, void *d_out, void *d_in, uint32_t lg_domain_size,
                                     uint32_t lg_blowup, size_t width, void *stream);
RustError sppark_b200_ntt_matrix(int field, size_t device_id, void *inout, uint32_t lg_domain_size,
                                 size_t width, int ntt_order, int ntt_direction, int ntt_type);

/* ---- polynomial helpers (SURVEY.md section 8, row f4) ----------------------------------------------
 * The reference's polynomial/ templates and ff/batch_inversion.hpp for the NTT fields above.  All
 * arrays are DEVICE memory in the field's memory format (the format compute_ntt uses), the work is
 * enqueued on `stream` and not synchronised; `len` is any size, not only a power of two.
 *   prefix_op          polynomial/prefix_op.cuh:322-384: inclusive prefix, op 0 = Add, 1 = Multiply;
 *                      d_out[i] = d_inp[0] (op) ... (op) d_inp[i]; d_out may be d_inp
 *   div_by_x_minus_z   polynomial/div_by_x_minus_z.cuh:445-486: divide c[0] + c[1] x + ... by (x - z)
 *                      in place; z is ONE element in HOST memory (the reference takes it by const
 *                      reference); rotate == 0: d_inout[0] = remainder, d_inout[1..] = quotient,
 *                      rotate != 0: d_inout[..len-2] = quotient, d_inout[len-1] = remainder
 *   evaluate           polynomial/evaluate.cuh:308-414: d_ret[k] = sum_i d_coeffs[i] * d_x[k]^i, k < n
 *   batch_inverse      ff/batch_inversion.hpp:14-51 over a whole array: d_out[i] = 1 / d_inp[i], and
 *                      zero where d_inp[i] is zero; d_out may be d_inp */
RustError sppark_b200_prefix_op_dev(int field, int op, void *d_out, const void *d_inp, size_t len, void *stream);
RustError sppark_b200_div_by_x_minus_z_dev(int field, void *d_inout, size_t len, const void *z, int rotate,
                                           void *stream);
RustError sppark_b200_evaluate_dev(int field, void *d_ret, const void *d_x, size_t n, const void *d_coeffs,
                                   size_t len, void *stream);
RustError sppark_b200_batch_inverse_dev(int field, void *d_out, const void *d_inp, size_t len, void *stream);

/* Slab-sharded NTT over G = 2^lg_g GPUs with ONE all-to-all (new; the reference has no multi-GPU
 * path).  N = N1 x N2, N1 = 2^ceil(lg/2).  Rank r owns input columns x[j1*N2 + j2],
 * j2 in [r*N2/G, (r+1)*N2/G), as a row-major [N1][N2/G] device array, and ends with the output
 * coefficients X[k1 + N1*k2], k1 in [r*N1/G, (r+1)*N1/G), as a row-major [N2][N1/G] array.
 *   which = 1: d_in = local input, d_out = staging buffer (N/G elements) laid out [G][N2/G][N1/G];
 *              then exchange block q with rank q (NCCL all-to-all, torch.distributed, ...)
 *   which = 2: d_in == d_out = the received buffer, transformed in place.
 * Both calls enqueue on `stream`.  sppark_b200/parallel.py: ntt_slab(). */
RustError sppark_b200_ntt_slab_pass(int field, int which, const void *d_in, void *d_out,
                                    uint32_t lg_domain_size, uint32_t lg_g, uint32_t rank,
                                    int ntt_direction, void *stream);

/* Fused exchange: stage 1 of the slab-sharded NTT storing every output row directly into the
 * receive buffer of the rank that owns it (NVLink peer memory) -- no staging buffer, no
 * all-to-all.  peer_recv[q], q < 2^lg_g (<= 8), = rank q's receive buffer of 2^(lg-lg_g)
 * elements as mapped into THIS process (sppark_b200_peer_open; peer_recv[rank] = the local
 * buffer).  The caller synchronises the ranks (any collective on `stream`) before stage 2
 * (sppark_b200_ntt_slab_pass, which = 2) reads its own buffer. */
RustError sppark_b200_ntt_slab_pass_p2p(int field, const void *d_in, void *const *peer_recv,
                                        uint32_t lg_domain_size, uint32_t lg_g, uint32_t rank,
                                        int ntt_direction, void *stream);
/* The same transform with every rank inside ONE process (a Rust / Go / C++ host needs no process
 * group): `inout` is a host array of 2^lg elements in natural order (order NN); chunk r runs on
 * device_ids[r], ndev = 1, 2, 4 or 8.  The exchange is fused into stage 1 (NVLink peer stores) when
 * the devices are distinct and can access each other, block copies otherwise. */
RustError sppark_b200_ntt_sharded(int field, void *inout, uint32_t lg_domain_size, int ntt_direction,
                                  const int *device_ids, size_t ndev);

/* Peer buffers (one process per GPU): cudaMalloc + CUDA IPC handle (64 bytes) on the owner,
 * cudaIpcOpenMemHandle / cudaIpcCloseMemHandle on the other ranks of the same node. */
RustError sppark_b200_peer_alloc(size_t bytes, void **d_ptr, void *ipc_handle_64);
RustError sppark_b200_peer_open(const void *ipc_handle_64, void **d_ptr);
RustError sppark_b200_peer_close(void *d_ptr);
RustError sppark_b200_peer_free(void *d_ptr);

/* Output on failure, for every entry that returns Jacobian points (mult_pippenger*, the MSM entries
 * below and sppark_b200_msm_combine): once the size of the output is known -- the curve id is valid (for
 * the _ctx_invoke entries: the context is not null) and batch * jacobian_bytes fits a size_t --, every
 * failure sets all output points to infinity (all-zero), refusals of bad arguments included.  An unknown
 * curve or a null context leaves the output as it was.  Bad arguments are refused with
 * -cudaErrorInvalidValue.
 *
 * MSM on any supported curve with host pointers (mult_pippenger's signature + curve id;
 * the reference has no PoC boundary for Pasta, SURVEY.md section 8d config 4). */
RustError sppark_b200_msm(int curve, void *out_jacobian, const void *points_affine,
                          size_t npoints, const void *scalars, size_t ffi_affine_sz);
/* Same with the reference template's `mont` flag (msm/pippenger.cuh:730-733): scalars_mont != 0
 * means the scalars are Montgomery residues (the C++ default there; the crates pass false). */
RustError sppark_b200_msm_ex(int curve, void *out_jacobian, const void *points_affine,
                             size_t npoints, const void *scalars, size_t ffi_affine_sz,
                             int scalars_mont);
/* Same over small scalars: scalar i is the little-endian unsigned integer in bytes
 * [i * scalar_bytes, (i + 1) * scalar_bytes) (a u32, u64 or u128 array on a little-endian host, or the
 * 32-byte layout), scalar_bytes = 4, 8, 16 or 32; bits from nbits up are ignored, 1 <= nbits <=
 * min(255, 8 * scalar_bytes).  Plain integers, no Montgomery flag.  The MSM runs ceil((nbits + 1) / c)
 * windows instead of ceil(256 / c) and moves scalar_bytes per scalar; nbits = 255 with 32-byte scalars
 * is sppark_b200_msm_ex(..., 0). */
RustError sppark_b200_msm_bits(int curve, void *out_jacobian, const void *points_affine, size_t npoints,
                               const void *scalars, size_t ffi_affine_sz, uint32_t scalar_bytes, uint32_t nbits);
/* One MSM sharded by point-chunk over GPUs of this process (SURVEY.md section 8e): chunk i of the points /
 * scalars runs on device_ids[i] through the host-pointer pipeline of that device, the ndev partial
 * results are added on the first device.  ndev = 1..64; ids may repeat (chunks of one device run
 * one after the other).  The multi-process route (one rank per GPU, NCCL all-gather of the
 * partials) is sppark_b200/parallel.py. */
RustError sppark_b200_msm_sharded(int curve, void *out_jacobian, const void *points_affine, size_t npoints,
                                  const void *scalars, size_t ffi_affine_sz, int scalars_mont,
                                  const int *device_ids, size_t ndev);
/* Preloaded points: the reference's msm_t{points, npoints} constructor + invoke(out, scalars)
 * (msm/pippenger.cuh:377-390,582-601) -- a fixed SRS stays on the device (of the calling thread's
 * current GPU), each invoke moves only the scalars (host pointer; npoints <= preloaded count). */
typedef struct sppark_b200_msm_ctx sppark_b200_msm_ctx;
RustError sppark_b200_msm_ctx_create(int curve, const void *points_affine, size_t npoints,
                                     size_t ffi_affine_sz, sppark_b200_msm_ctx **out);
/* Preloaded points as a precomputed fixed-base table: up to `copies` shifted copies 2^(c*V*k) * P_i
 * are stored, so that an invoke needs V = ceil(D/K) bucket sets instead of D windows (DESIGN.md
 * section 5a).  copies = 1 is sppark_b200_msm_ctx_create.  Fails for copies = 0 and for
 * copies * npoints >= 2^31.  _invoke and _free serve both kinds of context. */
RustError sppark_b200_msm_ctx_create_precomputed(int curve, const void *points_affine, size_t npoints,
                                                 size_t ffi_affine_sz, uint32_t copies,
                                                 sppark_b200_msm_ctx **out);
RustError sppark_b200_msm_ctx_invoke(sppark_b200_msm_ctx *ctx, void *out_jacobian, const void *scalars,
                                     size_t npoints, int scalars_mont);
/* _invoke over small scalars (format as sppark_b200_msm_bits).  A precomputed table keeps its width c
 * and bucket sets V; only the digits below ceil((nbits + 1) / c), and so only the copies holding them,
 * are read. */
RustError sppark_b200_msm_ctx_invoke_bits(sppark_b200_msm_ctx *ctx, void *out_jacobian, const void *scalars,
                                          size_t npoints, uint32_t scalar_bytes, uint32_t nbits);
void      sppark_b200_msm_ctx_free(sppark_b200_msm_ctx *ctx);
/* msm_t::invoke with device-resident points and scalars (msm/pippenger.cuh:582-601):
 * d_points: packed affine {X,Y}; d_scalars: 32-B LE; result written to HOST out_jacobian
 * after synchronising `stream`. */
RustError sppark_b200_msm_dev(int curve, void *out_jacobian, const void *d_points,
                              size_t npoints, const void *d_scalars, void *stream);
/* sppark_b200_msm_dev over small scalars (format as sppark_b200_msm_bits); d_scalars must be aligned
 * to min(scalar_bytes, 16) bytes, each scalar is read with one load of its width. */
RustError sppark_b200_msm_dev_bits(int curve, void *out_jacobian, const void *d_points, size_t npoints,
                                   const void *d_scalars, uint32_t scalar_bytes, uint32_t nbits, void *stream);
/* Batched MSM: B = batch scalar vectors of npoints scalars each, against one point set, in one call.
 * Vector b is the scalars [b * npoints, (b + 1) * npoints) in the small-scalar format of
 * sppark_b200_msm_bits (scalar_bytes = 4, 8, 16 or 32, plain integers -- not Montgomery form --,
 * bits from nbits up ignored; 32 and 255 for full-width scalars).  out_jacobians: HOST array of batch
 * Jacobian points (batch * jacobian_bytes); result b is the same group element as the single entry
 * with vector b.  The vectors run in groups that share one sort, accumulate, reduce and finish.
 * batch == 0 is a no-op; npoints == 0 gives batch points at infinity.  A bad format, npoints past the
 * context's count, batch * npoints * scalar_bytes overflowing size_t or misaligned device scalars are
 * refused before any device work.
 *   _ctx_invoke_batch: host scalars against the first npoints preloaded points of a plain or
 *     precomputed context; the scalars of the next group are uploaded while a group computes.
 *   _dev_batch: device points and scalars (aligned as for sppark_b200_msm_dev_bits); the work runs on
 *     `stream`, which is synchronised before return. */
RustError sppark_b200_msm_ctx_invoke_batch(sppark_b200_msm_ctx *ctx, void *out_jacobians, const void *scalars,
                                           size_t npoints, size_t batch, uint32_t scalar_bytes, uint32_t nbits);
RustError sppark_b200_msm_dev_batch(int curve, void *out_jacobians, const void *d_points, size_t npoints,
                                    const void *d_scalars, size_t batch, uint32_t scalar_bytes, uint32_t nbits,
                                    void *stream);
/* Scalar multiplication of point arrays: out[i] = s_i * P_i for i < npoints, as packed affine {X, Y} rows
 * (affine_bytes each, infinity = (0, 0)) -- the format sppark_b200_msm_ctx_create and mult_pippenger take.
 * Scalars use the format of sppark_b200_msm_bits: scalar_bytes = 4, 8, 16 or 32, plain integers (not
 * Montgomery form); bits from nbits up are ignored.  s_i is taken as an integer, not reduced mod r.
 * One lane per point runs a signed 5-bit window ladder (DESIGN.md section 5e); it is not constant-time.
 *   _dev: device memory, enqueued on `stream` without a synchronisation.  d_out == d_points (in place) is
 *     allowed, any other overlap of the output with the inputs is refused; d_scalars aligned as for
 *     sppark_b200_msm_dev_bits.
 *   host entry: input rows as sppark_b200_msm reads them (ffi_affine_sz 0: packed rows; larger: rows with
 *     an infinity flag after Y); the output is packed rows.  Synchronised before return.
 * An unknown curve, a bad scalar format, a null pointer with npoints > 0, npoints >= 2^31, a partial
 * overlap, misaligned device scalars or a bad host stride is refused with -cudaErrorInvalidValue before
 * any device work, the output untouched.  npoints == 0 is a no-op. */
RustError sppark_b200_scale_points_dev(int curve, void *d_out, const void *d_points, size_t npoints,
                                       const void *d_scalars, uint32_t scalar_bytes, uint32_t nbits,
                                       void *stream);
RustError sppark_b200_scale_points(int curve, void *out_affine, const void *points_affine, size_t npoints,
                                   const void *scalars, size_t ffi_affine_sz, uint32_t scalar_bytes,
                                   uint32_t nbits);

/* synthetic inputs: d_out[i] = (i+1)*G as packed affine points in DEVICE memory (the role of
 * util::generate_points_scalars, poc/msm-cuda/src/util.rs:11-38); enqueued on `stream`. */
RustError sppark_b200_generate_points_dev(int curve, void *d_out, size_t n, void *stream);
/* sum of `count` Jacobian points (host arrays): combines per-GPU partial MSM results after the
 * all-gather of a sharded MSM (NCCL cannot add curve points). */
RustError sppark_b200_msm_combine(int curve, void *out_jacobian, const void *partials, size_t count);

/* device self-test hook for the known-answer tests: r[i] = a[i] (op) b[i] through the PTX field
 * arithmetic; field 0 = BLS12-381 fp (48 B), 1 = BLS12-381 fr, 2 = Pallas fp, 3 = Vesta fp
 * (32 B each); op 0 mul (Montgomery), 1 add, 2 sub, 3 sqr, 4 mul_shared, 5 sqr_shared,
 * 6 msub_shared(a, b, b, a^2), 7 msub_shared with four operands: a = (a_i, c_i), b = (b_i, d_i)
 * interleaved (2n elements each), r[i] = a_i*b_i - c_i*d_i.  Host arrays. */
RustError sppark_b200_selftest_field(int field, int op, size_t n, void *r, const void *a, const void *b);
/* same for the single-word NTT fields (SPPARK_FIELD_GL64: 8-byte words, SPPARK_FIELD_BB31: 4-byte
 * Montgomery words): op 0 mul (Goldilocks: b is a canonical constant in Montgomery form, the result
 * a*b*2^-64 mod p, see csrc/ff/gl64.cuh), 1 add, 2 sub (b canonical), 3 tight, 4 canon. */
RustError sppark_b200_selftest_word_field(int field, int op, size_t n, void *r, const void *a, const void *b);
/* device self-test hook for the MSM's bucket sort: n host scalars (8 little-endian 32-bit words
 * each), window width wbits (3..24), cap entries per bin-sort CTA (0 = default; smaller values
 * send more bins down the overflow path).  Host outputs: counts and offsets per (window, bucket)
 * slot (nwins << (wbits - 1) each), the sorted entries (nwins * n), one slot per heavy bucket, and
 * info = {nwins, heavy threshold, #heavy buckets, log2 bins per window, #overflow bins}. */
RustError sppark_b200_selftest_msm_sort(size_t n, uint32_t wbits, uint32_t cap, const void *scalars, void *counts,
                                        void *offsets, void *sorted, void *heavy_slots, uint32_t *info);

/* introspection */
size_t      sppark_b200_ngpus(void);               /* ngpus(), util/gpu_t.cuh:21 */
int         sppark_b200_sm_count(int device_id);
const char *sppark_b200_version(void);
/* number of kernels this library has launched since load (bench.py's gpu_launches) */
uint64_t    sppark_b200_launch_count(void);
/* phase timing of the LAST MSM / NTT call with CUDA events on the call's own stream (the
 * roofline leg of bench.py): enable, run, synchronise, read (name, ms) pairs. */
void        sppark_b200_profile_enable(int on);
int         sppark_b200_profile_read(const char **names, float *ms, int cap);

#ifdef __cplusplus
}
#endif
#endif
