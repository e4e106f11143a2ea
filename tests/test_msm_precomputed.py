"""Precomputed fixed-base MSM contexts on the CPU (csrc/msm/msm_core.cuh make_config_precomputed /
digit_slot, csrc/msm/msm_table.cuh): the chooser table, and the CPU single-stepper
tests/emu/msm_precomputed_emu.cpp -- the table built by the same HD bodies as on the device, then
the whole pipeline with the digit -> (bucket set, copy) mapping -- compared with the oracle."""
import ctypes as C
import random

import numpy as np
import pytest

from test_emu import R_BLS, _build, _scalars

FIELDS = ("wbits", "nwins", "lg_nb", "npoints", "heavy", "heavy_chunk", "merge", "copies", "copy_stride", "digits")


@pytest.fixture(scope="module")
def emu():
    l = _build("msm_precomputed_emu")
    for fn in (l.emu_precomputed_bls12_381, l.emu_precomputed_pallas):
        fn.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_uint, C.c_uint, C.c_uint,
                       C.c_uint, C.c_uint, C.c_void_p]
    l.emu_config.argtypes = [C.c_size_t, C.c_uint, C.c_void_p]
    return l


@pytest.fixture
def clean_env(monkeypatch):
    for k in ("SPPARK_B200_MSM_WBITS", "SPPARK_B200_MSM_HEAVY"):
        monkeypatch.delenv(k, raising=False)
    return monkeypatch


def _config(emu, n, copies):
    out = np.zeros(10, dtype=np.uint32)
    emu.emu_config(n, copies, out.ctypes.data)
    return dict(zip(FIELDS, (int(v) for v in out)))


def _model(n, K):
    """the cost model of make_config_precomputed, in Python"""
    best = None
    for c in range(4, 25):
        D = -(-256 // c)
        V = -(-D // K)
        cost = 1.11 * D * n + 5.5 * V * 2 ** (c - 1)
        if best is None or cost < best[0]:
            best = (cost, c)
    return best[1]


# ---- the chooser ---------------------------------------------------------------------------------
def test_chooser_table(emu, clean_env):
    for lg in range(10, 29):
        n = 1 << lg
        plain = _config(emu, n, 0)
        assert _config(emu, n, 1) == plain, lg                      # K = 1: make_config, field for field
        assert plain["copies"] == 1 and plain["digits"] == plain["nwins"] and plain["copy_stride"] == n
        for K in range(1, plain["digits"] + 1):
            cfg = _config(emu, n, K)
            if K == 1:
                continue
            c, V, Ku, D = cfg["wbits"], cfg["nwins"], cfg["copies"], cfg["digits"]
            assert 4 <= c <= 24 and c == _model(n, K), (lg, K, cfg)
            assert D == -(-256 // c) and cfg["lg_nb"] == c - 1
            assert V == -(-D // K) and V * Ku >= D and (Ku - 1) * V < D and 2 <= Ku <= K, (lg, K, cfg)
            assert cfg["copy_stride"] == n and cfg["npoints"] == n and cfg["merge"] == 0
            assert cfg["heavy"] == min(max(D * n // 57000, 256), 16384), (lg, K, cfg)
            assert cfg["heavy_chunk"] == min(max(4 * cfg["heavy"], 2048), 16384)


def test_chooser_issue_examples(emu, clean_env):
    """the configurations the cost model ranks first at the sizes DESIGN.md section 5a tabulates"""
    got = {(lg, K): (_config(emu, 1 << lg, K)["wbits"], _config(emu, 1 << lg, K)["nwins"]) for lg, K in
           [(16, 16), (20, 4), (20, 14), (22, 13), (26, 4), (26, 6)]}
    assert got == {(16, 16): (16, 1), (20, 4): (16, 4), (20, 14): (19, 1), (22, 13): (20, 1),
                   (26, 4): (22, 3), (26, 6): (24, 2)}


def test_chooser_honours_width_override(emu, clean_env):
    for c in (3, 7, 24):
        clean_env.setenv("SPPARK_B200_MSM_WBITS", str(c))
        for K in (2, 5, 100):
            cfg = _config(emu, 1 << 18, K)
            D = -(-256 // c)
            assert cfg["wbits"] == c and cfg["nwins"] == -(-D // min(K, D)), (c, K, cfg)
    clean_env.setenv("SPPARK_B200_MSM_WBITS", "25")                # out of range: ignored
    assert _config(emu, 1 << 18, 4)["wbits"] == _model(1 << 18, 4)


# ---- the pipeline over a table ----------------------------------------------------------------------
def _inputs(oracle, curve, n, c, seed):
    """points: 61 distinct ones repeated, infinity at row 3, row 8 = -row 7; scalars: uniform, with r - 1,
    every digit +2^(c-1), a run of equal scalars (heavy buckets) and equal scalars on rows 7 and 8"""
    nl = 6 if curve == "bls12_381" else 4
    p = oracle.ff_consts(curve + "_fp")["p"]
    r = R_BLS if curve == "bls12_381" else oracle.ff_consts("vesta_fp")["p"]     # Pallas' group order
    base = oracle.gen_points(curve, 61)
    pts = base[np.arange(n) % 61].copy()
    if n > 3:
        pts[3] = 0
    if n > 8:
        y = sum(int(v) << (64 * i) for i, v in enumerate(pts[7][nl:]))
        pts[8][:nl] = pts[7][:nl]
        pts[8][nl:] = [((p - y) >> (64 * i)) & (2**64 - 1) for i in range(nl)]
    rnd = random.Random(seed)
    vals = [rnd.randrange(r) for _ in range(n)]
    D = -(-256 // c)
    top = sum((1 << (c - 1)) << (c * w) for w in range(D) if c * w + c - 1 < 255)
    for k, v in enumerate([r - 1, top, (1 << 255) - 1]):
        if k < n:
            vals[(k * 97 + 1) % n] = v
    if n > 8:
        vals[8] = vals[7]
    if n >= 100:
        vals[n // 2: n // 2 + n // 4] = [vals[n // 2]] * (n // 4)
    return pts, _scalars(vals)


def _emu_run(emu, curve, pts, sc, m, c, K, heavy=0, nslices=1, chunk=0):
    nl = 6 if curve == "bls12_381" else 4
    fn = emu.emu_precomputed_bls12_381 if curve == "bls12_381" else emu.emu_precomputed_pallas
    out, info = np.zeros(3 * nl, dtype=np.uint64), np.zeros(5, dtype=np.uint32)
    fn(out.ctypes.data, pts.ctypes.data, pts.shape[0], sc.ctypes.data, m, c, K, heavy, nslices, chunk, info.ctypes.data)
    return out, [int(v) for v in info]


def _reference(oracle, curve, pts, sc):
    return oracle.jac_to_affine(curve, oracle.msm(curve, pts, sc, "pippenger", ncpus=4))


def _check(oracle, emu, curve, pts, sc, m, c, K, **kw):
    want = _reference(oracle, curve, pts[:m], sc[:m])
    out, info = _emu_run(emu, curve, pts, sc, m, c, K, **kw)
    D = -(-256 // c)
    assert info[:4] == [c, -(-D // min(K, D)), D, -(-D // -(-D // min(K, D)))], (c, K, info)
    assert np.array_equal(oracle.jac_to_affine(curve, out), want), (curve, pts.shape[0], m, c, K, kw)


@pytest.mark.parametrize("curve", ["bls12_381", "pallas"])
@pytest.mark.parametrize("n", [1, 2, 33, 1000])
@pytest.mark.parametrize("c", [3, 4, 5, 8, 13])
def test_pipeline_over_table(oracle, emu, clean_env, curve, n, c):
    pts, sc = _inputs(oracle, curve, n, c, n * 31 + c)
    for K in (1, 2, 3, -(-256 // c)):
        _check(oracle, emu, curve, pts, sc, n, c, K, chunk=max(1, n // 3))


@pytest.mark.parametrize("curve,c,K", [("bls12_381", 8, 32), ("bls12_381", 13, 2), ("pallas", 5, 3), ("pallas", 4, 64)])
def test_pipeline_over_table_5000(oracle, emu, clean_env, curve, c, K):
    pts, sc = _inputs(oracle, curve, 5000, c, c * K)
    _check(oracle, emu, curve, pts, sc, 5000, c, K, chunk=1200)


@pytest.mark.parametrize("curve", ["bls12_381", "pallas"])
@pytest.mark.parametrize("c,K,nslices,heavy", [(5, 2, 3, 0), (8, 32, 4, 0), (4, 3, 2, 20), (13, 20, 5, 3), (3, 86, 7, 0)])
def test_prefixes_and_slices_shorter_than_the_copy_stride(oracle, emu, clean_env, curve, c, K, nslices, heavy):
    """an invoke of m < N scalars cut into slices: slice s reads rows [first, first + n) of every
    copy, the copies N rows apart; heavy thresholds forced low so that slices merge heavy buckets"""
    n = 700
    pts, sc = _inputs(oracle, curve, n, c, 7 * c + nslices)
    for m in (n, 451, 1):
        _check(oracle, emu, curve, pts, sc, m, c, K, heavy=heavy, nslices=nslices, chunk=97)


def test_pipeline_default_width_and_all_infinity(oracle, emu, clean_env):
    """the chooser's own width (make_config_precomputed) for a few K; a point set of infinities only"""
    pts, sc = _inputs(oracle, "bls12_381", 300, 8, 5)
    want = _reference(oracle, "bls12_381", pts, sc)
    for K in (1, 2, 4, 64):
        out, info = _emu_run(emu, "bls12_381", pts, sc, 300, 0, K, chunk=64)
        assert np.array_equal(oracle.jac_to_affine("bls12_381", out), want), (K, info)
    zero = np.zeros_like(pts)
    out, _ = _emu_run(emu, "bls12_381", zero, sc, 300, 6, 43, chunk=50)
    assert not out.any()
