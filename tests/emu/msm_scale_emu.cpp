// CPU single-stepper for scale_points -- TEST INFRASTRUCTURE ONLY.
// Runs the HD bodies of sppark_b200/csrc/msm/msm_scale.cuh in chunks, as msm::scale_points launches
// them: the ladder per point, pair_invert_body over the chunk's ZZZ, normalize_to_row per point.
// Not linked into the product.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <algorithm>
#include <vector>
#include "../../sppark_b200/csrc/ff/fields.cuh"
#include "../../sppark_b200/csrc/msm/msm_scale.cuh"

using namespace msm;

template<class F, uint32_t SW>
static void ladder(const uint32_t* points, const uint32_t* scalars, uint32_t nbits, uint32_t n, uint32_t* xyzz,
                   uint32_t* zzz)
{
    for (uint32_t i = 0; i < n; i++) scale_ladder_body<F, SW>(points, scalars, nbits, xyzz, zzz, i);
}

// out = n packed affine rows; scalars of scalar_bytes each; chunk 0: SCALE_CHUNK
template<class F>
static void emu_scale(uint32_t* out, const uint32_t* points, size_t npoints, const uint8_t* scalars,
                      uint32_t scalar_bytes, uint32_t nbits, size_t chunk)
{
    if (chunk == 0) chunk = SCALE_CHUNK;
    const uint32_t SW = scalar_bytes / 4;
    std::vector<uint32_t> xyzz, zzz;
    for (size_t first = 0; first < npoints; first += chunk) {
        const uint32_t n = (uint32_t)std::min(chunk, npoints - first);
        xyzz.assign((size_t)n * 4 * F::N, 0xdeadbeef);
        zzz.assign((size_t)n * F::N, 0xdeadbeef);
        const uint32_t* p = points + first * 2 * F::N;
        const uint32_t* s = reinterpret_cast<const uint32_t*>(scalars + first * scalar_bytes);
        switch (SW) {
        case 1: ladder<F, 1>(p, s, nbits, n, xyzz.data(), zzz.data()); break;
        case 2: ladder<F, 2>(p, s, nbits, n, xyzz.data(), zzz.data()); break;
        case 4: ladder<F, 4>(p, s, nbits, n, xyzz.data(), zzz.data()); break;
        default: ladder<F, 8>(p, s, nbits, n, xyzz.data(), zzz.data()); break;
        }
        for (uint32_t tid = 0; tid * PAIR_M < n; tid++) pair_invert_body<F>(zzz.data(), n, tid);
        for (uint32_t i = 0; i < n; i++)
            normalize_to_row<F>(xyzz.data(), zzz.data(), i, out + (first + i) * 2 * F::N);
    }
}

extern "C" void emu_scale_bls12_381(uint32_t* out, const uint32_t* points, size_t n, const uint8_t* scalars,
                                    uint32_t scalar_bytes, uint32_t nbits, size_t chunk)
{   emu_scale<ff::bls12_381_fp_t>(out, points, n, scalars, scalar_bytes, nbits, chunk);   }
extern "C" void emu_scale_pallas(uint32_t* out, const uint32_t* points, size_t n, const uint8_t* scalars,
                                 uint32_t scalar_bytes, uint32_t nbits, size_t chunk)
{   emu_scale<ff::pallas_fp_t>(out, points, n, scalars, scalar_bytes, nbits, chunk);   }
