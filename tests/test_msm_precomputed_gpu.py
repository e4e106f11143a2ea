"""Precomputed fixed-base MSM contexts on the device (MsmContext(curve, points, precompute=K),
sppark_b200_msm_ctx_create_precomputed): every curve against the reference, the debug line against
the chooser (make_config_precomputed / config_for_table, compiled with g++ here), forced widths,
special scalars and heavy buckets, the two-slice resident schedule, and the error paths.

Inputs and references are those of test_msm_geometry_gpu.py: m distinct points repeated (point INF
infinity, point NEG = -(NEG - 1)), the reference being the m-point MSM with the scalars folded per
point mod r."""
import os
import re
import subprocess

import numpy as np
import pytest

from test_msm_geometry_gpu import INF, R_BLS, _curve, _fold, _int, _limbs, _mixed, _need_device_bytes, _uniform

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CFG_SRC = r'''
#include <cstdio>
#include <cstdlib>
#include <algorithm>
#include "sppark_b200/csrc/msm/msm_core.cuh"
// argv: N K m -> the geometry an invoke of m scalars runs on a context of N points built with K:
// "wbits sets digits copies heavy heavy_chunk"
int main(int argc, char** argv)
{
    const size_t N = strtoull(argv[1], nullptr, 10), m = strtoull(argv[3], nullptr, 10);
    const uint32_t K = (uint32_t)atoi(argv[2]);
    const msm::Config t = msm::make_config_precomputed(N, K);
    const msm::Config c = t.copies == 1 ? msm::make_config(m) : msm::config_for_table(m, t.wbits, t.copies, N);
    printf("%u %u %u %u %u %u\n", c.wbits, c.nwins, msm::digit_count(c), c.copies, c.heavy, c.heavy_chunk);
    return 0;
}
'''
LINE = re.compile(r"\[msm\] slice (\d+) n=(\d+) wbits=(\d+) nwins=(\d+) heavy_thr=(\d+) tasks_claimed=\d+ "
                  r"nheavy=(\d+) nchunks=(\d+) acc_blocks=\d+ digits=(\d+) sets=(\d+) copies=(\d+)")
CURVES = ["bls12_381", "pallas", "vesta", "bn254", "bls12_377", "bls12_381_g2", "bn254_g2", "bls12_377_g2"]
ROW_BYTES = {"bls12_381": 96, "pallas": 64, "vesta": 64, "bn254": 64, "bls12_377": 96, "bls12_381_g2": 192,
             "bn254_g2": 128, "bls12_377_g2": 192}
FR = {"bls12_381": "bls12_381_fr", "pallas": "vesta_fp", "vesta": "pallas_fp", "bn254": "bn254_fr",
      "bls12_377": "bls12_377_fr", "bls12_381_g2": "bls12_381_fr", "bn254_g2": "bn254_fr", "bls12_377_g2": "bls12_377_fr"}


@pytest.fixture(scope="module")
def cfg_exe(tmp_path_factory):
    d = tmp_path_factory.mktemp("precomputed")
    src, exe = d / "cfg.cpp", d / "cfg"
    src.write_text(CFG_SRC)
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-I", ROOT, "-I", "/usr/local/cuda/include", "-o", str(exe), str(src)])
    return str(exe)


def _geometry(exe, N, K, m):
    """the chooser's geometry under the current environment"""
    v = list(map(int, subprocess.check_output([exe, str(N), str(K), str(m)], text=True).split()))
    return dict(zip(("wbits", "sets", "digits", "copies", "heavy", "heavy_chunk"), v))


@pytest.fixture
def debug(monkeypatch, capfd):
    monkeypatch.setenv("SPPARK_B200_MSM_DEBUG", "1")
    for k in ("SPPARK_B200_MSM_WBITS", "SPPARK_B200_MSM_HEAVY", "SPPARK_B200_MSM_SLICES",
              "SPPARK_B200_MSM_SCHED", "SPPARK_B200_MSM_PAIR"):
        monkeypatch.delenv(k, raising=False)
    capfd.readouterr()
    return capfd


def _lines(err):
    return [tuple(map(int, t)) for t in LINE.findall(err)]


def _check_lines(err, exe, N, K, m, nslices=1):
    """one debug line per slice, each with the chooser's width, sets, digits, copies and threshold"""
    g = _geometry(exe, N, K, m)
    lines = _lines(err)
    assert len(lines) == nslices, err[-2000:]
    for line in lines:
        assert (line[2], line[3], line[4], line[7], line[8], line[9]) == \
            (g["wbits"], g["sets"], g["heavy"], g["digits"], g["sets"], g["copies"]), (line, g)
    return lines


def _k_single_set(exe, N):
    """K = D of the width that K = D itself selects: one bucket set, no Horner step"""
    K = _geometry(exe, N, 64, N)["digits"]
    assert _geometry(exe, N, K, N)["sets"] == 1
    return K


def _ctx(cv, rows, K):
    from sppark_b200 import msm
    return msm.MsmContext(cv.cid, rows, precompute=K)


def _arkworks(pts, m):
    nl = pts.shape[1]
    ark = np.zeros((pts.shape[0], nl + 1), dtype=np.uint64)
    ark[:, :nl] = pts
    ark[INF::m, :nl] = 7                                # a flagged row's coordinates are ignored
    ark[INF::m, nl] = 1
    return ark


# ---- every curve -----------------------------------------------------------------------------------
@pytest.mark.parametrize("curve", CURVES)
def test_every_curve(oracle, debug, cfg_exe, curve):
    """packed and arkworks rows, prefixes N / 1000 / 1, Montgomery-form scalars, K = 1, 2 and D"""
    cv = _curve(oracle, curve)
    m = 32 if cv.g2py is not None else 256
    N = 4099
    base = cv.base(m)
    pts = np.ascontiguousarray(np.resize(base, (N, base.shape[1])))
    sc = _mixed(N, 5 + cv.cid, 12, cv.r, m)
    mont = np.array([_limbs(oracle.ff_op(FR[curve], "to_mont", _int(row) % cv.r)) for row in sc[:1000]], dtype=np.uint64)
    refs = {n: cv.reference(base, _fold(sc[:n], m, cv.r)) for n in (N, 1000, 1)}
    for K in (1, 2, _k_single_set(cfg_exe, N)):
        for rows in (pts, _arkworks(pts, m)):
            ctx = _ctx(cv, rows, K)
            try:
                for n in (N, 1000, 1):
                    debug.readouterr()
                    got = ctx.invoke(np.ascontiguousarray(sc[:n]))
                    _check_lines(debug.readouterr().err, cfg_exe, N, K, n)
                    assert cv.affine(got) == refs[n], (curve, K, rows.shape, n)
                got = ctx.invoke(mont, mont=True)
                assert cv.affine(got) == cv.reference(base, _fold(np.array([_limbs(_int(r) % cv.r) for r in sc[:1000]],
                                                                           dtype=np.uint64), m, cv.r)), (curve, K, "mont")
            finally:
                ctx.close()


@pytest.mark.parametrize("curve", ["bls12_381", "bls12_381_g2"])
def test_one_copy_is_the_plain_context(oracle, debug, curve):
    """precompute=1 runs the plain context's geometry and returns its point.  (Jacobian limbs are not
    compared: the order of the entries inside a bucket is set by atomics, so the representative of
    the point varies from call to call, for any context.)"""
    from sppark_b200 import msm
    cv = _curve(oracle, curve)
    base = cv.base(256)
    pts = np.ascontiguousarray(np.resize(base, (20000, base.shape[1])))
    sc = _uniform(20000, 8, r=cv.r)
    a, b = msm.MsmContext(cv.cid, pts), msm.MsmContext(cv.cid, pts, precompute=1)
    try:
        for n in (20000, 777):
            debug.readouterr()
            got_a = a.invoke(sc[:n].copy())
            la = [line[2:] for line in _lines(debug.readouterr().err)]
            got_b = b.invoke(sc[:n].copy())
            lb = [line[2:] for line in _lines(debug.readouterr().err)]
            assert la == lb and la[0][-1] == 1, (la, lb)
            assert cv.affine(got_a) == cv.affine(got_b) == cv.reference(base, _fold(sc[:n], 256, cv.r)), n
    finally:
        a.close()
        b.close()


# ---- forced widths -----------------------------------------------------------------------------------
@pytest.mark.parametrize("curve,c", [("bls12_381", c) for c in range(3, 25)] + [("pallas", c) for c in range(3, 21)])
def test_forced_width(oracle, debug, monkeypatch, cfg_exe, curve, c):
    """SPPARK_B200_MSM_WBITS at every value it accepts, K = 4 (V = ceil(D/4) sets, every set full width)"""
    monkeypatch.setenv("SPPARK_B200_MSM_WBITS", str(c))
    cv = _curve(oracle, curve)
    N, K = 4099, 4
    g = _geometry(cfg_exe, N, K, N)
    bucket = 2 * ROW_BYTES[curve]
    _need_device_bytes((g["sets"] << (c - 1)) * bucket + (1 << 30))
    base = cv.base(512)
    pts = np.ascontiguousarray(np.resize(base, (N, base.shape[1])))
    sc = _mixed(N, c, c, cv.r, 512)
    ctx = _ctx(cv, pts, K)
    try:
        debug.readouterr()
        got = ctx.invoke(sc)
        _check_lines(debug.readouterr().err, cfg_exe, N, K, N)
    finally:
        ctx.close()
    assert cv.affine(got) == cv.reference(base, _fold(sc, 512, cv.r))


# ---- special scalars and heavy buckets ---------------------------------------------------------------
@pytest.mark.parametrize("K", [2, 3, 16])
def test_special_scalars_and_heavy_buckets(oracle, debug, cfg_exe, K):
    """2^17 points: the special scalars of every width mixed in, and 3000 rows of one scalar plus
    bucket runs planted in digit sets other than 0 (heavy buckets, the cooperative kernels)"""
    cv = _curve(oracle, "bls12_381")
    N = 1 << 17
    g = _geometry(cfg_exe, N, K, N)
    c = g["wbits"]
    sc = _mixed(N, 40 + K, c, R_BLS, 512)
    sc[1000:4000] = sc[1000]
    for k, b in enumerate((3, 40, 41)):
        sc[5000 + 700 * k: 5700 + 700 * k] = _limbs((b + 1) << (c * (g["digits"] - 2 - k)))
    base = cv.base(512)
    pts = np.ascontiguousarray(np.resize(base, (N, 12)))
    ctx = _ctx(cv, pts, K)
    try:
        debug.readouterr()
        got = ctx.invoke(sc)
        lines = _check_lines(debug.readouterr().err, cfg_exe, N, K, N)
    finally:
        ctx.close()
    assert lines[0][5] > 0, "no heavy bucket: the heavy kernels did not run"
    assert cv.affine(got) == cv.reference(base, _fold(sc, 512, R_BLS))


# ---- two resident slices ----------------------------------------------------------------------------------
@pytest.mark.parametrize("K", [2, 4])
def test_two_slice_schedule_2pow22(oracle, debug, cfg_exe, K):
    """2^22 + 4096 points: invokes of >= 2^22 scalars run as two slices (N/8, rest), the second one
    reading rows [first, ...) of every copy; 2^22 - 1 scalars run as one"""
    cv = _curve(oracle, "bls12_381")
    m, N = 512, (1 << 22) + 4096
    g = _geometry(cfg_exe, N, K, N)
    entries = g["sets"] * g["copies"] * N
    _need_device_bytes(g["copies"] * N * 96 + N * 32 + entries * 12 + (g["sets"] << (g["wbits"] - 1)) * 192 + (2 << 30))
    base = cv.base(m)
    pts = np.resize(base, (N, 12))
    sc = _mixed(N, 22 + K, g["wbits"], R_BLS, m)
    ctx = _ctx(cv, pts, K)
    try:
        for n in (N, 1 << 22, (1 << 22) - 1):
            debug.readouterr()
            got = ctx.invoke(np.ascontiguousarray(sc[:n]))
            _check_lines(debug.readouterr().err, cfg_exe, N, K, n, nslices=2 if n >= 1 << 22 else 1)
            assert cv.affine(got) == cv.reference(base, _fold(sc[:n], m, R_BLS)), (K, n)
    finally:
        ctx.close()


# ---- errors --------------------------------------------------------------------------------------------
def test_error_paths(oracle):
    from sppark_b200 import _lib, msm
    cv = _curve(oracle, "bls12_381")
    pts = np.ascontiguousarray(cv.base(1000))
    with pytest.raises(_lib.SpparkError, match="copies"):
        msm.MsmContext(cv.cid, pts, precompute=0)
    with pytest.raises(_lib.SpparkError, match="2\\^31"):
        msm.MsmContext(cv.cid, pts, precompute=-(-(1 << 31) // 1000))          # K * N >= 2^31
    ctx = msm.MsmContext(cv.cid, pts, precompute=-(-(1 << 31) // 1000) - 1)   # K * N < 2^31: K clamped to D
    try:
        with pytest.raises(_lib.SpparkError, match="more scalars"):
            ctx.invoke(_uniform(1001, 1, r=R_BLS))
        sc = _uniform(1000, 2, r=R_BLS)
        assert cv.affine(ctx.invoke(sc)) == cv.reference(pts, sc)
    finally:
        ctx.close()
