"""GPU parity for the BLS12-381 G2 MSM (mult_pippenger_fp2_inf, poc/msm-cuda/cuda/
pippenger_inf.cu:36-47) through the C-ABI vs the CPU oracle (oracle/ec2.c) and vs the golden
vectors recorded from the reference's own CUDA build.  Compared as group elements
(affine-normalised), like poc/msm-cuda/tests/msm.rs:41-63 (msm_fp2_correctness, 2^14 points)."""
import os
import random

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

R_BLS = 0x73eda753299d7d483339d80809a1d80553bda402fffe5bfeffffffff00000001
G2 = 3


def _limbs(x, n=4):
    return [(x >> (64 * i)) & 0xFFFFFFFFFFFFFFFF for i in range(n)]


def _scalars(n, seed):
    rnd = random.Random(seed)
    return np.array([_limbs(rnd.randrange(R_BLS)) for _ in range(n)], dtype=np.uint64).reshape(n, 4)


def _ark(pts):
    a = np.zeros((pts.shape[0], 25), dtype=np.uint64)
    a[:, :24] = pts
    return a


def _same(oracle, a, b):
    return np.array_equal(oracle.g2_jac_to_affine(a), oracle.g2_jac_to_affine(b))


@pytest.mark.parametrize("n", [1, 2, 31, 33, 193, 1000, 4096])
def test_g2_msm_matches_oracle(oracle, n):
    from sppark_b200 import msm
    base = oracle.g2_points(min(n, 256))
    pts = _ark(base[np.arange(n) % base.shape[0]])
    if n > 3:
        pts[3, 24] = 1                               # flagged infinity (util.rs:29-31 plants one)
    sc = _scalars(n, n)
    got = msm.multi_scalar_mult_fp2_arkworks(pts, sc)
    want = oracle.g2_msm(pts, sc)
    assert _same(oracle, got, want)


@pytest.mark.parametrize("kind", ["zero", "one", "r_minus_1", "all_same", "pm_pairs", "coord_zero_inf"])
def test_g2_msm_adversarial(oracle, kind):
    from sppark_b200 import msm
    n = 600
    base = oracle.g2_points(64)
    pts = _ark(base[np.arange(n) % 64])
    sc = _scalars(n, 5)
    if kind == "zero":
        sc[:] = 0
    elif kind == "one":
        sc[:] = _limbs(1)
    elif kind == "r_minus_1":
        sc[:] = _limbs(R_BLS - 1)
    elif kind == "all_same":
        pts[:] = pts[7]
        sc[:] = sc[7]
    elif kind == "pm_pairs":                          # k*P + (r-k)*P cancels inside the buckets
        pts[1::2] = pts[0::2]
        for i in range(0, n, 2):
            k = sum(int(v) << (64 * j) for j, v in enumerate(sc[i]))
            sc[i + 1] = _limbs(R_BLS - k)
    else:
        pts[10:20, :24] = 0                           # X == Y == 0, flag clear
    got = msm.multi_scalar_mult_fp2_arkworks(pts, sc)
    want = oracle.g2_msm(pts, sc)
    assert _same(oracle, got, want)
    if kind in ("zero", "pm_pairs"):
        assert not got[24:].any()                     # Z == 0: infinity


def test_g2_msm_2pow14_folded(oracle):
    """The size of the reference's msm_fp2_correctness test; 2^14 points = 2^8 distinct points
    replicated, so the oracle checks it as a 256-point MSM with scalars folded mod r."""
    from sppark_b200 import msm
    n, m = 1 << 14, 1 << 8
    base = oracle.g2_points(m)
    pts = _ark(np.tile(base, (n // m, 1)))
    sc = _scalars(n, 14)
    got = msm.multi_scalar_mult_fp2_arkworks(pts, sc)
    ints = [0] * m
    for i in range(n):
        ints[i % m] += sum(int(v) << (64 * j) for j, v in enumerate(sc[i]))
    folded = np.array([_limbs(v % R_BLS) for v in ints], dtype=np.uint64)
    want = oracle.g2_msm(base, folded)
    assert _same(oracle, got, want)


def test_g2_packed_dev_generate_combine(oracle):
    import torch
    from sppark_b200 import msm
    d_pts = msm.generate_points_dev(G2, 200)
    pts = d_pts.cpu().numpy().view(np.uint64)
    assert np.array_equal(pts, oracle.g2_points(200))
    n = 5000
    idx = np.arange(n) % 200
    sc = _scalars(n, 9)
    want = oracle.g2_msm(pts[idx], sc)
    got = msm.msm(G2, np.ascontiguousarray(pts[idx]), sc)                       # packed host layout
    assert _same(oracle, got, want)
    got = msm.msm_dev(G2, d_pts[torch.from_numpy(idx).cuda()].contiguous(),
                      torch.from_numpy(sc.view(np.int64)).cuda())
    assert _same(oracle, got, want)
    parts = np.stack([msm.msm(G2, np.ascontiguousarray(pts[idx[k::2]]), np.ascontiguousarray(sc[k::2])) for k in range(2)])
    assert _same(oracle, msm.combine(G2, parts), want)


def test_g2_matches_reference_gpu_golden(oracle):
    """Same group element as the reference's own mult_pippenger_fp2_inf / mult_pippenger_inf
    recorded from its CUDA build (tests/golden/make_golden.py g2)."""
    from sppark_b200 import msm
    path = os.path.join(os.path.dirname(__file__), "golden", "msm_g2_ref_gpu.npz")
    if not os.path.exists(path):
        pytest.skip("G2 golden not recorded")
    g = np.load(path)
    for k in range(int(g["ncases"])):
        got = msm.multi_scalar_mult_fp2_arkworks(np.ascontiguousarray(g[f"points{k}"]), np.ascontiguousarray(g[f"scalars{k}"]))
        assert _same(oracle, got, g[f"out{k}"]), k
    for k in range(int(g["g1_ncases"])):
        got = msm.multi_scalar_mult_arkworks(np.ascontiguousarray(g[f"g1_points{k}"]), np.ascontiguousarray(g[f"g1_scalars{k}"]))
        assert np.array_equal(oracle.jac_to_affine("bls12_381", got), oracle.jac_to_affine("bls12_381", g[f"g1_out{k}"])), k
