"""CPU: the G2 oracle (oracle/ec2.c) against an independent big-integer model and against the
golden vectors recorded from the reference's mult_pippenger_fp2_inf on a GPU."""
import os
import random

import numpy as np
import pytest

P = 0x1a0111ea397fe69a4b1ba7b6434bacd764774b84f38512bf6730d2a0f6b0f6241eabfffeb153ffffb9feffffffffaaab
R_BLS = 0x73eda753299d7d483339d80809a1d80553bda402fffe5bfeffffffff00000001
MONT = 1 << 384
HERE = os.path.dirname(os.path.abspath(__file__))


def to_limbs(x, n=6):
    return [(x >> (64 * i)) & (2**64 - 1) for i in range(n)]


def from_limbs(a):
    return sum(int(v) << (64 * i) for i, v in enumerate(a))


def f2_enc(c):
    return np.array(to_limbs(c[0] * MONT % P) + to_limbs(c[1] * MONT % P), dtype=np.uint64)


def f2_dec(a):
    rinv = pow(MONT, -1, P)
    return (from_limbs(a[:6]) * rinv % P, from_limbs(a[6:12]) * rinv % P)


def f2_mul(a, b):
    return ((a[0] * b[0] - a[1] * b[1]) % P, (a[0] * b[1] + a[1] * b[0]) % P)


def f2_inv(a):
    d = pow(a[0] * a[0] + a[1] * a[1], -1, P)
    return (a[0] * d % P, -a[1] * d % P)


def aff_add(p, q):
    """Affine chord-and-tangent over Fp2 (None = infinity): the textbook group law."""
    if p is None:
        return q
    if q is None:
        return p
    if p[0] == q[0]:
        if (p[1][0] + q[1][0]) % P == 0 and (p[1][1] + q[1][1]) % P == 0:
            return None
        x2 = f2_mul(p[0], p[0])
        lam = f2_mul(((3 * x2[0]) % P, (3 * x2[1]) % P), f2_inv(((2 * p[1][0]) % P, (2 * p[1][1]) % P)))
    else:
        lam = f2_mul(((q[1][0] - p[1][0]) % P, (q[1][1] - p[1][1]) % P),
                     f2_inv(((q[0][0] - p[0][0]) % P, (q[0][1] - p[0][1]) % P)))
    l2 = f2_mul(lam, lam)
    x3 = ((l2[0] - p[0][0] - q[0][0]) % P, (l2[1] - p[0][1] - q[0][1]) % P)
    t = f2_mul(lam, ((p[0][0] - x3[0]) % P, (p[0][1] - x3[1]) % P))
    return (x3, ((t[0] - p[1][0]) % P, (t[1] - p[1][1]) % P))


def aff_mul(p, k):
    acc = None
    while k:
        if k & 1:
            acc = aff_add(acc, p)
        p = aff_add(p, p)
        k >>= 1
    return acc


def pt_dec(xy):
    x, y = f2_dec(xy[:12]), f2_dec(xy[12:24])
    return None if x == (0, 0) and y == (0, 0) else (x, y)


def sc_arr(vals):
    return np.array([to_limbs(v, 4) for v in vals], dtype=np.uint64)


def test_fp2_ops_vs_python(oracle):
    rng = random.Random(11)
    a = [(rng.randrange(P), rng.randrange(P)) for _ in range(20)] + [(0, 0), (1, 0), (0, 1), (P - 1, P - 1)]
    b = [(rng.randrange(P), rng.randrange(P)) for _ in range(len(a))]
    A, B = np.stack([f2_enc(x) for x in a]), np.stack([f2_enc(x) for x in b])
    for op, fn in [("mul", f2_mul), ("add", lambda x, y: ((x[0] + y[0]) % P, (x[1] + y[1]) % P)),
                   ("sub", lambda x, y: ((x[0] - y[0]) % P, (x[1] - y[1]) % P))]:
        got = oracle.fp2_op(op, A, B)
        for i in range(len(a)):
            assert f2_dec(got[i]) == fn(a[i], b[i]), op
    got = oracle.fp2_op("sqr", A)
    inv = oracle.fp2_op("inv", A[:20])
    for i in range(len(a)):
        assert f2_dec(got[i]) == f2_mul(a[i], a[i])
    for i in range(20):
        assert f2_dec(inv[i]) == f2_inv(a[i])


def test_g2_generator_and_points(oracle):
    pts = oracle.g2_points(20)
    g = pt_dec(pts[0])
    # IETF pairing-friendly-curves, BLS12-381 G2 generator, x.c0
    assert g[0][0] == 0x024aa2b2f08f0a91260805272dc51051c6e47ad4fa403b02b4510b647ae3d1770bac0326a805bbefd48056c8c121bdb8
    acc = None
    for i in range(20):
        acc = aff_add(acc, g)
        assert pt_dec(pts[i]) == acc
        assert oracle.g2_on_curve(pts[i])
    bad = pts[3].copy()
    bad[0] ^= np.uint64(1)
    assert not oracle.g2_on_curve(bad)


def test_g2_group_order(oracle):
    pts = oracle.g2_points(3)
    for k, want_inf in [(R_BLS, True), (R_BLS - 1, False), (R_BLS + 1, False)]:
        r = oracle.g2_msm(pts[1:2], sc_arr([k % 2**256]), "naive")
        is_inf = not r[24:].any()
        assert is_inf == want_inf
    # (r-1)*P == -P
    r = oracle.g2_jac_to_affine(oracle.g2_msm(pts[1:2], sc_arr([R_BLS - 1]), "naive"))
    p = pt_dec(pts[1])
    assert pt_dec(r) == (p[0], ((-p[1][0]) % P, (-p[1][1]) % P))


@pytest.mark.parametrize("n", [1, 7, 100])
def test_g2_naive_buckets_python_agree(oracle, n):
    rng = random.Random(n)
    base = oracle.g2_points(16)
    pts = base[[rng.randrange(16) for _ in range(n)]]
    ks = [rng.randrange(R_BLS) for _ in range(n)]
    ks[0] = R_BLS - 1
    a = oracle.g2_jac_to_affine(oracle.g2_msm(pts, sc_arr(ks), "naive"))
    b = oracle.g2_jac_to_affine(oracle.g2_msm(pts, sc_arr(ks), "buckets"))
    assert np.array_equal(a, b)
    if n <= 7:
        want = None
        for i in range(n):
            want = aff_add(want, aff_mul(pt_dec(pts[i]), ks[i]))
        assert pt_dec(a) == want


def test_g2_infinity_inputs(oracle):
    base = oracle.g2_points(4)
    ark = np.zeros((4, 25), dtype=np.uint64)
    ark[:, :24] = base
    ark[2, 24] = 1                       # flagged infinity, coordinates left in place
    ks = sc_arr([5, 6, 7, 8])
    got = oracle.g2_jac_to_affine(oracle.g2_msm(ark, ks))
    want = oracle.g2_jac_to_affine(oracle.g2_msm(base[[0, 1, 3]], sc_arr([5, 6, 8])))
    assert np.array_equal(got, want)
    zero = base.copy()
    zero[1] = 0                          # X == Y == 0 is infinity too
    got = oracle.g2_jac_to_affine(oracle.g2_msm(zero, ks))
    want = oracle.g2_jac_to_affine(oracle.g2_msm(base[[0, 2, 3]], sc_arr([5, 7, 8])))
    assert np.array_equal(got, want)
    # cancellation: k*P + (r-k)*P = inf
    got = oracle.g2_msm(base[[1, 1]], sc_arr([12345, R_BLS - 12345]))
    assert not got[24:].any()


def test_g2_oracle_matches_reference_gpu_golden(oracle):
    path = os.path.join(HERE, "golden", "msm_g2_ref_gpu.npz")
    if not os.path.exists(path):
        pytest.skip("G2 golden not recorded")
    g = np.load(path)
    for k in range(int(g["ncases"])):
        pts, sc, want = g[f"points{k}"], g[f"scalars{k}"], g[f"out{k}"]
        got = oracle.g2_jac_to_affine(oracle.g2_msm(pts, sc))
        assert np.array_equal(got, oracle.g2_jac_to_affine(want)), k
        assert oracle.g2_on_curve(oracle.g2_jac_to_affine(want))
    # the arkworks-layout G1 entry point of the same reference build
    for k in range(int(g["g1_ncases"])):
        pts = g[f"g1_points{k}"].copy()
        pts[pts[:, 12] != 0, :12] = 0
        got = oracle.jac_to_affine("bls12_381", oracle.msm("bls12_381", np.ascontiguousarray(pts[:, :12]), g[f"g1_scalars{k}"]))
        assert np.array_equal(got, oracle.jac_to_affine("bls12_381", g[f"g1_out{k}"])), k


def test_reference_fp2_inf_entry_is_inconsistent(oracle):
    """Documents why the pin above is taken on packed points (oracle/ref_msm_g2.cu): the reference's
    own mult_pippenger_fp2_inf, as built with nvcc, agrees with its packed instantiation only for
    n = 1; for n = 2 it returns s0*P0 (point 1 is read at the wrong pitch and taken for infinity)."""
    path = os.path.join(HERE, "golden", "msm_g2_ref_gpu.npz")
    if not os.path.exists(path):
        pytest.skip("G2 golden not recorded")
    g = np.load(path)
    same = [np.array_equal(oracle.g2_jac_to_affine(g[f"inf_out{k}"]), oracle.g2_jac_to_affine(g[f"out{k}"]))
            for k in range(int(g["ncases"]))]
    assert same[0] and not any(same[1:])
    s0p0 = oracle.g2_jac_to_affine(oracle.g2_msm(g["points1"][:1], g["scalars1"][:1]))
    assert np.array_equal(oracle.g2_jac_to_affine(g["inf_out1"]), s0p0)
