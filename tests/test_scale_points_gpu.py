"""Scalar multiplication of point arrays on the device (sppark_b200_scale_points[_dev], csrc/msm/msm_scale.cuh)
on every curve, against a plain reference of every product s * P as an affine point: the C oracle for G1
and BLS12-381 G2, oracle/g2py.py for BN254 and BLS12-377 G2.

Inputs repeat m distinct points (one at infinity, one the negative of its neighbour) against a cycle of
k scalars with m and k coprime, so each product is computed once by the reference.  At 2^20 points
the result is checked independently through the MSM: sum_i 1 * out_i == sum_i s_i * P_i."""
import numpy as np
import pytest

from test_msm_geometry_gpu import _curve, _int, _limbs, INF

pytestmark = pytest.mark.gpu

CURVES = ["bls12_381", "pallas", "vesta", "bn254", "bls12_377", "bls12_381_g2", "bn254_g2", "bls12_377_g2"]
NL = {"bls12_381": 6, "pallas": 4, "vesta": 4, "bn254": 4, "bls12_377": 6, "bls12_381_g2": 12, "bn254_g2": 8,
      "bls12_377_g2": 12}
W = 5                   # msm::SCALE_WBITS


def _special(r, nbits=255):
    half = 1 << (W - 1)
    return [0, 1, 2, half, half + 1, (1 << nbits) - 1, r - 1, r, r + 1, (1 << 255) - 1,
            sum((half + 1) << (W * w) for w in range(64) if W * w + W <= nbits)]


class Products:
    """the reference s * P of one curve, memoised per (point row, scalar)"""

    def __init__(self, oracle, name):
        self.cv, self.oracle, self.name, self.memo = _curve(oracle, name), oracle, name, {}

    def one(self, row, k):
        """the device takes k as an integer; the test points lie in the subgroup of order r, so k mod r
        gives the same point (the C oracle reads only the bits of r's length)"""
        key = (row.tobytes(), k)
        if key not in self.memo:
            cv, o, nl = self.cv, self.oracle, NL[self.name]
            k %= cv.r
            if cv.g2py is not None:
                R = cv.g2py.smul(k, cv.g2py.decode_affine(row)[0]) if row.any() else None
                self.memo[key] = cv.g2py.encode_affine([R])[0]
            else:
                sc = np.array([_limbs(k)], dtype=np.uint64)
                if self.name == "bls12_381_g2":
                    jac = o.g2_msm(row[None], sc, "naive")
                    self.memo[key] = o.g2_jac_to_affine(jac) if jac.any() else np.zeros(2 * nl, np.uint64)
                else:
                    jac = o.msm(self.name, row[None], sc, "naive")
                    self.memo[key] = o.jac_to_affine(self.name, jac) if jac.any() else np.zeros(2 * nl, np.uint64)
        return self.memo[key]

    def rows(self, pts, vals):
        return np.stack([self.one(pts[i], v) for i, v in enumerate(vals)])


def _inputs(oracle, name, n, nbits=255, sbytes=32, m=29, seed=0):
    """n rows of m distinct points and a cycle of k scalars (the special values of nbits, then random
    ones; garbage above nbits); returns points, the raw scalar bytes (n, sbytes) and the values mod 2^nbits"""
    cv = _curve(oracle, name)
    rng = np.random.default_rng(seed)
    cyc = [v % (1 << nbits) for v in _special(cv.r, nbits)]
    cyc += [int.from_bytes(rng.bytes(32), "little") % (1 << nbits) for _ in range(6)]
    while np.gcd(len(cyc), m) != 1:
        cyc.append(int.from_bytes(rng.bytes(32), "little") % (1 << nbits))
    pts = cv.base(m)[np.arange(n) % m].copy()
    vals = [cyc[i % len(cyc)] for i in range(n)]
    raw = rng.integers(0, 256, size=(n, sbytes), dtype=np.uint8)            # garbage above nbits
    low = np.frombuffer(((1 << nbits) - 1).to_bytes(sbytes, "little"), dtype=np.uint8)
    vb = np.frombuffer(b"".join(v.to_bytes(sbytes, "little") for v in vals), dtype=np.uint8).reshape(n, sbytes)
    raw = (raw & ~low) | (vb & low)
    return pts, raw, vals


def _host_scalars(raw):
    sb = raw.shape[1]
    flat = np.ascontiguousarray(raw).reshape(-1)
    if sb == 4:
        return flat.view(np.uint32).copy()
    if sb == 8:
        return flat.view(np.uint64).copy()
    return flat.view(np.uint64).reshape(-1, sb // 8).copy()


def _dev_scalars(raw):
    import torch
    h = _host_scalars(raw)
    return torch.from_numpy(h.view(np.int32 if h.dtype == np.uint32 else np.int64)).cuda()


def _dev_points(pts):
    import torch
    return torch.from_numpy(np.ascontiguousarray(pts).view(np.int64)).cuda()


def _host(t):
    import torch
    torch.cuda.synchronize()
    return t.cpu().numpy().view(np.uint64)


@pytest.mark.parametrize("name", CURVES)
@pytest.mark.parametrize("n", [1, 2, 31, 33, 1000, (1 << 16) + 3])
def test_device_entry(oracle, name, n):
    from sppark_b200 import msm
    ref = Products(oracle, name)
    pts, raw, vals = _inputs(oracle, name, n, seed=n)
    got = _host(msm.scale_points_dev(_curve(oracle, name).cid, _dev_points(pts), _dev_scalars(raw)))
    assert np.array_equal(got, ref.rows(pts, vals)), (name, n)
    if n > INF:
        assert not got[INF].any()


@pytest.mark.parametrize("name", ["bls12_381", "pallas", "bn254_g2"])
@pytest.mark.parametrize("sbytes,nbits", [(4, 1), (4, 31), (8, 8), (8, 64), (16, 100), (16, 128), (32, 128), (32, 255)])
def test_scalar_formats(oracle, name, sbytes, nbits):
    from sppark_b200 import msm
    ref = Products(oracle, name)
    n = 300
    pts, raw, vals = _inputs(oracle, name, n, nbits, sbytes, seed=sbytes * 1000 + nbits)
    cid = _curve(oracle, name).cid
    got = _host(msm.scale_points_dev(cid, _dev_points(pts), _dev_scalars(raw), nbits=nbits))
    assert np.array_equal(got, ref.rows(pts, vals)), (name, sbytes, nbits)
    got = msm.scale_points(cid, pts, _host_scalars(raw), nbits=nbits)
    assert np.array_equal(got, ref.rows(pts, vals)), (name, sbytes, nbits)


@pytest.mark.parametrize("name", ["bls12_381", "bls12_381_g2"])
def test_forced_chunks_and_in_place(oracle, name, monkeypatch):
    """chunks of 1000 points, n across three boundaries; the device entry in place"""
    from sppark_b200 import msm
    monkeypatch.setenv("SPPARK_B200_SCALE_CHUNK", "1000")
    ref = Products(oracle, name)
    n = 3017
    pts, raw, vals = _inputs(oracle, name, n, seed=5)
    want = ref.rows(pts, vals)
    cid = _curve(oracle, name).cid
    d = _dev_points(pts)
    assert np.array_equal(_host(msm.scale_points_dev(cid, d, _dev_scalars(raw))), want)
    out = msm.scale_points_dev(cid, d, _dev_scalars(raw), out=d)
    assert out.data_ptr() == d.data_ptr() and np.array_equal(_host(d), want)
    assert np.array_equal(msm.scale_points(cid, pts, _host_scalars(raw)), want)


@pytest.mark.parametrize("pinned", [False, True])
def test_host_entry_row_layouts(oracle, pinned):
    """packed rows and 104-byte arkworks rows (flag word after Y: a flagged row is infinity whatever its
    coordinates), from pinned and pageable memory"""
    import torch
    from sppark_b200 import msm
    ref = Products(oracle, "bls12_381")
    n = 2000
    pts, raw, vals = _inputs(oracle, "bls12_381", n, seed=11)
    flags = np.zeros(n, dtype=np.uint64)
    flags[7::50] = 1
    ark = np.concatenate([pts, flags[:, None]], axis=1)
    ark[flags == 1, :12] = pts[3]                               # coordinates of a real point, flagged away
    packed_want = ref.rows(pts, vals)
    want = packed_want.copy()
    want[flags == 1] = 0
    sc = _host_scalars(raw)
    if pinned:
        def pin(a):
            t = torch.empty(a.shape, dtype=torch.int64 if a.dtype == np.uint64 else torch.int32, pin_memory=True)
            v = t.numpy().view(a.dtype)
            v[...] = a
            return v
        pts, ark, sc = pin(pts), pin(ark), pin(sc)
    assert np.array_equal(msm.scale_points(msm.BLS12_381_G1, pts, sc), packed_want)
    assert ark.strides[0] == 104
    assert np.array_equal(msm.scale_points(msm.BLS12_381_G1, ark, sc), want)


def test_side_stream(oracle):
    import torch
    from sppark_b200 import msm
    ref = Products(oracle, "pallas")
    pts, raw, vals = _inputs(oracle, "pallas", 4000, seed=3)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        d, sc = _dev_points(pts), _dev_scalars(raw)
        out = msm.scale_points_dev(msm.PALLAS, d, sc, stream=s.cuda_stream)
    s.synchronize()
    assert np.array_equal(out.cpu().numpy().view(np.uint64), ref.rows(pts, vals))


@pytest.mark.parametrize("name,lg", [("bls12_381", 20), ("bn254", 20), ("bls12_381_g2", 18)])
def test_large_through_the_msm(oracle, name, lg):
    """sum_i 1 * out_i == sum_i s_i * P_i (two device MSMs); a seeded sample of 512 rows against the
    reference, every one of them on the curve"""
    import torch
    from sppark_b200 import msm
    cv = _curve(oracle, name)
    n = 1 << lg
    d = msm.generate_points_dev(cv.cid, n)
    g = torch.Generator(device="cpu").manual_seed(lg)
    sc = torch.randint(-2**63, 2**63 - 1, (n, 4), dtype=torch.int64, generator=g).cuda()
    out = msm.scale_points_dev(cv.cid, d, sc)
    ones = torch.ones(n, dtype=torch.int32, device="cuda")
    lhs = msm.msm_dev(cv.cid, out, ones, nbits=1)
    rhs = msm.msm_dev(cv.cid, d, sc)
    assert cv.affine(lhs) == cv.affine(rhs), name
    idx = np.random.default_rng(lg).choice(n, 512, replace=False)
    pts, got = _host(d)[idx], _host(out)[idx]
    sch = _host(sc)[idx]
    ref = Products(oracle, name)
    vals = [_int(r) % (1 << 255) for r in sch]
    assert np.array_equal(got, ref.rows(pts, vals)), name
    for row in got:
        if name == "bls12_381_g2":
            assert oracle.g2_on_curve(row)
        else:
            assert oracle.on_curve(name, row)
