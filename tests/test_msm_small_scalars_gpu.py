"""MSM over small scalars on the device: 4-, 8-, 16- and 32-byte scalars with a bit bound, through the
host (pageable and pinned), device-tensor and preloaded entries, on every curve.

The reference is the oracle on the scalars reduced mod 2^nbits (every bit above nbits is random here,
and must be ignored).  Large inputs repeat m distinct points, so the reference is the m-point MSM of
the folded scalars, as in test_msm_geometry_gpu.py.  With SPPARK_B200_MSM_DEBUG=1 every slice prints
its geometry; the cases check that it ran the window count the bound gives and the scalar format."""
import re

import numpy as np
import pytest

from test_msm_geometry_gpu import _curve, _fold, _schedule

LINE = re.compile(r"\[msm\] slice (\d+) n=(\d+) wbits=(\d+) nwins=(\d+) heavy_thr=\d+ .*? digits=(\d+) sets=\d+ "
                  r"copies=(\d+) nbits=(\d+) sbytes=(\d+)")
G1 = ["pallas", "vesta", "bn254", "bls12_377"]
G2 = ["bls12_381_g2", "bn254_g2", "bls12_377_g2"]


@pytest.fixture
def debug(monkeypatch, capfd):
    monkeypatch.setenv("SPPARK_B200_MSM_DEBUG", "1")
    for k in ("SPPARK_B200_MSM_WBITS", "SPPARK_B200_MSM_HEAVY", "SPPARK_B200_MSM_SLICES",
              "SPPARK_B200_MSM_SCHED", "SPPARK_B200_MSM_PAIR"):
        monkeypatch.delenv(k, raising=False)
    capfd.readouterr()
    return capfd


# ---- scalars --------------------------------------------------------------------------------------
def _raw(n, sbytes, seed):
    return np.random.default_rng(seed).integers(0, 256, size=(n, sbytes), dtype=np.uint8)


def _array(raw):
    """the host array msm() takes for scalars of raw.shape[1] bytes"""
    sb = raw.shape[1]
    flat = np.ascontiguousarray(raw).reshape(-1)
    if sb == 4:
        return flat.view(np.uint32).copy()
    if sb == 8:
        return flat.view(np.uint64).copy()
    return flat.view(np.uint64).reshape(-1, sb // 8).copy()


def _rows(raw, nbits):
    """(n, 4) uint64 rows of the scalars mod 2^nbits"""
    n, sb = raw.shape
    pad = np.zeros((n, 32), dtype=np.uint8)
    pad[:, :sb] = raw
    rows = pad.view(np.uint64).reshape(n, 4).copy()
    for k in range(4):
        keep = nbits - 64 * k
        if keep <= 0:
            rows[:, k] = 0
        elif keep < 64:
            rows[:, k] &= np.uint64((1 << keep) - 1)
    return rows


def _fill(n, sbytes, value, nbits, seed):
    """every scalar `value` below bit nbits, random bits from nbits up"""
    raw = _raw(n, sbytes, seed)
    low = np.frombuffer(((1 << nbits) - 1).to_bytes(sbytes, "little"), dtype=np.uint8)
    v = np.frombuffer(value.to_bytes(sbytes, "little"), dtype=np.uint8)
    return (raw & ~low) | (v & low)


def _width(nbits):
    return next(sb for sb in (4, 8, 16, 32) if nbits <= 8 * sb)


def _lines(err):
    return [tuple(map(int, t)) for t in LINE.findall(err)]


def _expect_geometry(lines, nbits, sbytes, nslices=1):
    assert len(lines) == nslices, lines
    for ln in lines:
        wbits, nwins, digits = ln[2], ln[3], ln[4]
        assert ln[6:] == (nbits, sbytes), ln
        assert digits == -(-(nbits + 1) // wbits), ln


def _host(cv, m, raw, nbits, debug, pts=None, pinned=False):
    from sppark_b200 import msm
    n = raw.shape[0]
    base = cv.base(m)
    if pts is None:
        pts = np.resize(base, (n, base.shape[1]))
    sc = _array(raw)
    if pinned:
        import torch
        t = torch.empty(sc.nbytes, dtype=torch.uint8).pin_memory()
        pinned_sc = t.numpy().view(sc.dtype).reshape(sc.shape)
        pinned_sc[...] = sc
        sc = pinned_sc
    debug.readouterr()
    got = msm.msm(cv.cid, pts, sc, nbits=nbits)
    lines = _lines(debug.readouterr().err)
    return got, lines, cv.reference(base, _fold(_rows(raw, nbits), m, cv.r))


# ---- the grid -----------------------------------------------------------------------------------------
GRID = [(1, 4), (2, 4), (8, 4), (16, 4), (31, 4), (32, 4), (33, 8), (63, 8), (64, 8), (65, 16), (100, 16),
        (128, 16), (129, 32), (200, 32), (254, 32), (255, 32)]


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 37, 5000])
@pytest.mark.parametrize("nbits,sbytes", GRID)
def test_bls12_381_grid(oracle, debug, nbits, sbytes, n):
    cv = _curve(oracle, "bls12_381")
    got, lines, want = _host(cv, 512, _raw(n, sbytes, nbits * 7 + n), nbits, debug)
    _expect_geometry(lines, nbits, sbytes)
    assert cv.affine(got) == want


@pytest.mark.gpu
@pytest.mark.parametrize("nbits", [1, 32, 64, 128, 255])
@pytest.mark.parametrize("curve", G1 + G2)
def test_other_curves(oracle, debug, curve, nbits):
    cv = _curve(oracle, curve)
    m = 32 if curve in ("bn254_g2", "bls12_377_g2") else 256
    sbytes = _width(nbits)
    got, lines, want = _host(cv, m, _raw(3000, sbytes, nbits + cv.cid), nbits, debug)
    _expect_geometry(lines, nbits, sbytes)
    assert cv.affine(got) == want


@pytest.mark.gpu
@pytest.mark.parametrize("nbits", [16, 64])
@pytest.mark.parametrize("c", [3, 8, 16, 24])
def test_forced_widths(oracle, debug, monkeypatch, c, nbits):
    """SPPARK_B200_MSM_WBITS: c = 8 and 16 divide both bounds (a top window holding only the carry)"""
    monkeypatch.setenv("SPPARK_B200_MSM_WBITS", str(c))
    cv = _curve(oracle, "bls12_381")
    got, lines, want = _host(cv, 512, _raw(4099, 8, c + nbits), nbits, debug)
    _expect_geometry(lines, nbits, 8)
    assert lines[0][2] == c and lines[0][3] == -(-(nbits + 1) // c)
    assert cv.affine(got) == want


@pytest.mark.gpu
@pytest.mark.parametrize("nbits", [1, 16, 64, 200])
def test_special_scalars(oracle, debug, nbits):
    """all zero below the bound (infinity), all 2^nbits - 1, one non-zero scalar"""
    cv = _curve(oracle, "bls12_381")
    sbytes, n = _width(nbits), 5000
    got, _, want = _host(cv, 512, _fill(n, sbytes, 0, nbits, 1), nbits, debug)
    assert not got.any() and want == cv.affine(got)
    got, _, want = _host(cv, 512, _fill(n, sbytes, (1 << nbits) - 1, nbits, 2), nbits, debug)
    assert cv.affine(got) == want
    one = np.zeros((n, sbytes), dtype=np.uint8)
    one[1234] = _raw(1, sbytes, 3)[0] | 1
    got, _, want = _host(cv, 512, one, nbits, debug)
    assert cv.affine(got) == want


@pytest.mark.gpu
@pytest.mark.parametrize("nbits,sbytes", [(1, 4), (16, 4), (32, 4), (64, 8), (100, 16), (200, 32)])
def test_pinned_host_and_device_tensors(oracle, debug, nbits, sbytes):
    import torch
    from sppark_b200 import msm
    cv = _curve(oracle, "bls12_381")
    n, m = 5000, 512
    raw = _raw(n, sbytes, nbits)
    got, lines, want = _host(cv, m, raw, nbits, debug, pinned=True)
    _expect_geometry(lines, nbits, sbytes)
    assert cv.affine(got) == want
    d_base = msm.generate_points_dev(cv.cid, m)
    dp = d_base.repeat(-(-n // m), 1)[:n].contiguous()
    base = d_base.cpu().numpy().view(np.uint64)
    sc = _array(raw)
    ds = torch.from_numpy(sc.view(np.int32 if sbytes == 4 else np.int64)).cuda()
    debug.readouterr()
    got = msm.msm_dev(cv.cid, dp, ds, nbits=nbits)
    _expect_geometry(_lines(debug.readouterr().err), nbits, sbytes)
    assert cv.affine(got) == cv.reference(base, _fold(_rows(raw, nbits), m, cv.r))


@pytest.mark.gpu
def test_misaligned_device_scalars_refused(oracle):
    """d_scalars must be aligned to min(scalar_bytes, 16): refused on the host, out set to infinity"""
    import torch
    from sppark_b200 import _lib, msm
    l = _lib.lib()
    dp = msm.generate_points_dev(msm.BLS12_381_G1, 16)
    ds = torch.zeros(256, dtype=torch.int32, device="cuda")
    for sbytes, off in ((8, 4), (16, 8), (32, 4), (32, 8)):
        out = np.ones(18, dtype=np.uint64)
        err = l.sppark_b200_msm_dev_bits(0, out.ctypes.data, dp.data_ptr(), 16, ds.data_ptr() + off, sbytes, 8,
                                         torch.cuda.current_stream().cuda_stream)
        code = err.code
        if err.message:
            l.drop_error_message(err.message)
        assert code == -1 and not out.any(), (sbytes, off)
    torch.cuda.synchronize()


@pytest.mark.gpu
@pytest.mark.parametrize("nbits", [1, 16, 64])
def test_plain_context_prefix(oracle, debug, nbits):
    """a plain preloaded context invoked on n < N points; the width follows (n, nbits)"""
    from sppark_b200 import msm
    cv = _curve(oracle, "bls12_381")
    N, n, m = 6000, 4097, 512
    base = cv.base(m)
    ctx = msm.MsmContext(cv.cid, np.resize(base, (N, 12)))
    try:
        sbytes = _width(nbits)
        raw = _raw(n, sbytes, nbits + 11)
        debug.readouterr()
        got = ctx.invoke(_array(raw), nbits=nbits)
        _expect_geometry(_lines(debug.readouterr().err), nbits, sbytes)
        assert cv.affine(got) == cv.reference(base, _fold(_rows(raw, nbits), m, cv.r))
    finally:
        ctx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("K", [4, 64])
def test_precomputed_context(oracle, debug, K):
    """K = 4 and K = D (every digit its own copy): the table keeps its width and sets, a bound below
    the table's reach reads only the first copies"""
    from sppark_b200 import msm
    cv = _curve(oracle, "bls12_381")
    N = 3000
    pts = cv.base(N)
    ctx = msm.MsmContext(cv.cid, pts, precompute=K)
    try:
        for nbits in (1, 16, 64, 128, 255):
            sbytes = _width(nbits)
            raw = _raw(N, sbytes, nbits + K)
            debug.readouterr()
            got = ctx.invoke(_array(raw), nbits=nbits)
            lines = _lines(debug.readouterr().err)
            _expect_geometry(lines, nbits, sbytes)
            assert cv.affine(got) == cv.reference(pts, _rows(raw, nbits)), (K, nbits)
    finally:
        ctx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("nbits", [1, 16, 64])
def test_slice_schedules(oracle, debug, nbits):
    """2^22 points: four slices on the host path, two on the resident path"""
    from sppark_b200 import msm
    cv = _curve(oracle, "bls12_381")
    n, m = 1 << 22, 512
    sbytes = _width(nbits)
    raw = _raw(n, sbytes, nbits + 22)
    want = cv.reference(cv.base(m), _fold(_rows(raw, nbits), m, cv.r))
    pts = np.resize(cv.base(m), (n, 12))
    sc = _array(raw)
    debug.readouterr()
    got = msm.msm(cv.cid, pts, sc, nbits=nbits)
    lines = _lines(debug.readouterr().err)
    _expect_geometry(lines, nbits, sbytes, len(_schedule(n)))
    assert [ln[1] for ln in lines] == _schedule(n)
    assert cv.affine(got) == want
    ctx = msm.MsmContext(cv.cid, pts)
    try:
        debug.readouterr()
        got = ctx.invoke(sc, nbits=nbits)
        lines = _lines(debug.readouterr().err)
        assert [ln[1] for ln in lines] == _schedule(n, resident=True)
        _expect_geometry(lines, nbits, sbytes, 2)
        assert cv.affine(got) == want
    finally:
        ctx.close()


@pytest.mark.gpu
def test_255_bits_is_todays_call(oracle, debug):
    """nbits = 255 with 32-byte scalars runs today's configuration through every entry: the same
    geometry on the debug line and the same point as msm_ex, msm_dev and ctx_invoke.  (The Jacobian
    limbs of one call are not unique: the order inside a bucket follows the sort's atomics, so the
    points are compared in affine normal form.)"""
    import torch
    from sppark_b200 import msm
    cv = _curve(oracle, "bls12_381")
    n, m = 20000, 512
    raw = _raw(n, 32, 255)
    raw[:, 31] &= 0x3f
    sc = _array(raw)
    base = cv.base(m)
    pts = np.resize(base, (n, 12))
    want = cv.reference(base, _fold(sc, m, cv.r))
    for k in (0, 1):
        debug.readouterr()
        got = msm.msm(cv.cid, pts, sc, nbits=255) if k else msm.msm(cv.cid, pts, sc)
        lines = _lines(debug.readouterr().err)
        assert cv.affine(got) == want
        if k:
            assert lines == old
        old = lines
    dp = torch.from_numpy(pts.view(np.int64)).cuda()
    ds = torch.from_numpy(sc.view(np.int64)).cuda()
    for k in (0, 1):
        debug.readouterr()
        got = msm.msm_dev(cv.cid, dp, ds, nbits=255) if k else msm.msm_dev(cv.cid, dp, ds)
        lines = [ln[2:] for ln in _lines(debug.readouterr().err)]
        assert cv.affine(got) == want
        if k:
            assert lines == old
        old = lines
    for K in (None, 4):
        ctx = msm.MsmContext(cv.cid, pts, precompute=K)
        try:
            for k in (0, 1):
                debug.readouterr()
                got = ctx.invoke(sc, nbits=255) if k else ctx.invoke(sc)
                lines = [ln[2:] for ln in _lines(debug.readouterr().err)]
                assert cv.affine(got) == want
                if k:
                    assert lines == old
                old = lines
        finally:
            ctx.close()
