"""Scalar multiplication of point arrays on the CPU: the CPU single-stepper tests/emu/msm_scale_emu.cpp
runs the HD bodies of csrc/msm/msm_scale.cuh (recode + ladder, pair inversion, normalise) chunk by
chunk, and every product is compared bit for bit with the oracle's naive s * P as an affine point;
then the argument checks of the two C entries, without a device."""
import ctypes as C
import random

import numpy as np
import pytest

from test_emu import R_BLS, _build

W = 5                                   # msm::SCALE_WBITS
INVAL, NODEV = -1, -100


@pytest.fixture(scope="module")
def emu():
    l = _build("msm_scale_emu")
    for fn in (l.emu_scale_bls12_381, l.emu_scale_pallas):
        fn.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_uint, C.c_uint, C.c_size_t]
    return l


def _order(oracle, curve):
    return R_BLS if curve == "bls12_381" else oracle.ff_consts("vesta_fp")["p"]


def _nl(curve):
    return 6 if curve == "bls12_381" else 4


def _points(oracle, curve, n):
    """distinct multiples of G with infinity at row 3, row 5 = row 4 (duplicate), row 8 = -row 7"""
    nl = _nl(curve)
    p = oracle.ff_consts(curve + "_fp")["p"]
    pts = oracle.gen_points(curve, 23)[np.arange(n) % 23].copy()
    if n > 3:
        pts[3] = 0
    if n > 5:
        pts[5] = pts[4]
    if n > 8:
        y = sum(int(v) << (64 * i) for i, v in enumerate(pts[7][nl:]))
        pts[8][:nl] = pts[7][:nl]
        pts[8][nl:] = [((p - y) >> (64 * i)) & (2**64 - 1) for i in range(nl)]
    return pts


def _pack(vals, sbytes):
    return np.frombuffer(b"".join(v.to_bytes(sbytes, "little") for v in vals), dtype=np.uint8).copy()


def _expected(oracle, curve, pts, vals, nbits):
    """rows of (v mod 2^nbits) * P by the oracle's naive MSM of one term"""
    out = np.zeros((len(vals), 2 * _nl(curve)), dtype=np.uint64)
    for i, v in enumerate(vals):
        v %= 1 << nbits
        row = np.array([[(v >> (64 * k)) & (2**64 - 1) for k in range(4)]], dtype=np.uint64)
        jac = oracle.msm(curve, pts[i:i + 1], row, "naive")
        out[i] = oracle.jac_to_affine(curve, jac) if jac.any() else 0
    return out


def _run(emu, curve, pts, vals, sbytes=32, nbits=255, chunk=0):
    out = np.full((pts.shape[0], 2 * _nl(curve)), 0xA5A5A5A5A5A5A5A5, dtype=np.uint64)
    sc = _pack(vals, sbytes) if vals else np.zeros(8, dtype=np.uint8)
    fn = emu.emu_scale_bls12_381 if curve == "bls12_381" else emu.emu_scale_pallas
    fn(out.ctypes.data, pts.ctypes.data, pts.shape[0], sc.ctypes.data, sbytes, nbits, chunk)
    return out


def _adversarial(r, nbits):
    half = 1 << (W - 1)
    vals = [0, 1, 2, half, half + 1, (1 << nbits) - 1, r - 1, r, r + 1, (1 << 255) - 1, (1 << W) - 1,
            sum((half + 1) << (W * w) for w in range(64) if W * w + W <= nbits),       # a carry into every window
            sum(half << (W * w) for w in range(64) if W * w + W <= nbits)]             # every digit +2^(w-1)
    return vals


@pytest.mark.parametrize("curve", ["bls12_381", "pallas"])
def test_adversarial_scalars(oracle, emu, curve):
    """every special scalar against every kind of point: infinity, duplicates, P next to -P"""
    r = _order(oracle, curve)
    special = _adversarial(r, 255)
    n = 3 * len(special)
    pts = _points(oracle, curve, n)
    rnd = random.Random(len(curve))
    # rows 0 .. n: each special value three times (against different points); garbage above bit 255
    vals = [special[i % len(special)] | (rnd.randrange(2) << 255) for i in range(n)]
    got = _run(emu, curve, pts, vals)
    want = _expected(oracle, curve, pts, vals, 255)
    assert np.array_equal(got, want)
    assert not got[3].any()                                    # infinity in, infinity out


@pytest.mark.parametrize("curve", ["bls12_381", "pallas"])
@pytest.mark.parametrize("sbytes,nbits", [(s, b) for s in (4, 8, 16, 32) for b in (1, 8, 31, 64, 100, 128, 255)
                                          if b <= 8 * s])
def test_scalar_formats(oracle, emu, curve, sbytes, nbits):
    """random words of every width with bits above nbits set; the special values of that bound"""
    rnd = random.Random(sbytes * 1000 + nbits)
    r = _order(oracle, curve)
    special = [v % (1 << (8 * sbytes)) for v in _adversarial(r, nbits)]
    vals = special + [rnd.randrange(1 << (8 * sbytes)) for _ in range(24)]
    pts = _points(oracle, curve, len(vals))
    got = _run(emu, curve, pts, vals, sbytes, nbits)
    assert np.array_equal(got, _expected(oracle, curve, pts, vals, nbits)), (sbytes, nbits)


@pytest.mark.parametrize("chunk", [1, 7, 64])
def test_chunks(oracle, emu, chunk):
    """chunks of the inversion that split the input anywhere, one of them shorter than the rest"""
    rnd = random.Random(chunk)
    n = 150
    pts = _points(oracle, "bls12_381", n)
    vals = [rnd.randrange(R_BLS) for _ in range(n)]
    vals[10] = 0
    got = _run(emu, "bls12_381", pts, vals, chunk=chunk)
    assert np.array_equal(got, _expected(oracle, "bls12_381", pts, vals, 255))


def test_no_points(emu):
    pts = np.zeros((0, 12), dtype=np.uint64)
    assert _run(emu, "bls12_381", pts, []).shape == (0, 12)


# ---- C ABI: argument checks, without a device ----------------------------------------------------------
def _no_gpu():
    import torch
    return not torch.cuda.is_available()


def _call(lib, name, *args):
    e = getattr(lib, name)(*args)
    msg = C.cast(e.message, C.c_char_p).value.decode() if e.message else None
    if e.message:
        lib.drop_error_message(e.message)
    return e.code, msg


class Bufs:
    """host buffers used as points, scalars and output (the checks never read them)"""

    def __init__(self):
        self.pts = np.arange(1, 1 + 13 * 8, dtype=np.uint64)
        self.sc = np.arange(500, 500 + 4 * 8, dtype=np.uint64)
        self.out = np.full(12 * 8 + 4, 7, dtype=np.uint64)
        self.keep = [a.copy() for a in (self.pts, self.sc, self.out)]

    def unchanged(self):
        return all(np.array_equal(a, b) for a, b in zip((self.pts, self.sc, self.out), self.keep))


DEV, HOST = "sppark_b200_scale_points_dev", "sppark_b200_scale_points"
FORMAT = ": scalar_bytes must be 4, 8, 16 or 32 and 1 <= nbits <= min(255, 8 * scalar_bytes)"
OVERLAP = ": the output may be the points (in place) but may not overlap them or the scalars otherwise"


def _dev(lib, u, curve=0, out=None, pts=None, n=4, sc=None, sbytes=32, nbits=255):
    out = u.out.ctypes.data if out is None else out
    pts = u.pts.ctypes.data if pts is None else pts
    sc = u.sc.ctypes.data if sc is None else sc
    return _call(lib, DEV, curve, out, pts, n, sc, sbytes, nbits, None)


def _host(lib, u, curve=0, out=None, pts=None, n=4, sc=None, ffi=0, sbytes=32, nbits=255):
    out = u.out.ctypes.data if out is None else out
    pts = u.pts.ctypes.data if pts is None else pts
    sc = u.sc.ctypes.data if sc is None else sc
    return _call(lib, HOST, curve, out, pts, n, sc, ffi, sbytes, nbits)


def test_unknown_curve(lib):
    u = Bufs()
    for c in (8, 9, -1):
        assert _dev(lib, u, curve=c) == (INVAL, DEV + ": unknown curve")
        assert _host(lib, u, curve=c) == (INVAL, HOST + ": unknown curve")
        assert _dev(lib, u, curve=c, n=0) == (INVAL, DEV + ": unknown curve")
    assert u.unchanged()


@pytest.mark.parametrize("sbytes,nbits", [(3, 8), (12, 8), (64, 8), (4, 0), (4, 33), (8, 65), (16, 129), (32, 256)])
def test_bad_scalar_format(lib, sbytes, nbits):
    u = Bufs()
    for curve in range(8):
        assert _dev(lib, u, curve=curve, sbytes=sbytes, nbits=nbits) == (INVAL, DEV + FORMAT)
        assert _host(lib, u, curve=curve, sbytes=sbytes, nbits=nbits) == (INVAL, HOST + FORMAT)
        assert _dev(lib, u, curve=curve, n=0, sbytes=sbytes, nbits=nbits) == (INVAL, DEV + FORMAT)
    assert u.unchanged()


def test_null_pointers_and_the_empty_call(lib):
    u = Bufs()
    for which in ("out", "pts", "sc"):
        kw = {which: None}
        # ctypes passes None as NULL: build the call by hand
        args = dict(out=u.out.ctypes.data, pts=u.pts.ctypes.data, sc=u.sc.ctypes.data)
        args.update(kw)
        assert (_call(lib, DEV, 0, args["out"], args["pts"], 4, args["sc"], 32, 255, None)
                == (INVAL, DEV + ": null pointer")), which
        assert (_call(lib, HOST, 0, args["out"], args["pts"], 4, args["sc"], 0, 32, 255)
                == (INVAL, HOST + ": null pointer")), which
        # npoints == 0: a no-op, whatever the pointers
        assert _call(lib, DEV, 0, args["out"], args["pts"], 0, args["sc"], 32, 255, None) == (0, None)
        assert _call(lib, HOST, 0, args["out"], args["pts"], 0, args["sc"], 0, 32, 255) == (0, None)
    assert _call(lib, HOST, 3, None, None, 0, None, 8, 8, 8) == (0, None)     # even a bad stride
    assert u.unchanged()


def test_too_many_points(lib):
    u = Bufs()
    for n in (1 << 31, (1 << 31) + 5, 1 << 40):
        assert _dev(lib, u, n=n) == (INVAL, DEV + ": npoints must be < 2^31")
        assert _host(lib, u, n=n) == (INVAL, HOST + ": npoints must be < 2^31")
    assert u.unchanged()


def test_partial_overlap(lib):
    u = Bufs()
    base = u.out.ctypes.data
    for curve, ab in ((0, 96), (1, 64), (3, 192)):
        n = 2
        # the output half over the points, the points inside the output, the scalars under the output
        for out, pts, sc in ((base, base + 48, u.sc.ctypes.data), (base + 16, base, u.sc.ctypes.data),
                             (base, u.pts.ctypes.data, base + ab), (base + 32, u.pts.ctypes.data, base)):
            assert _dev(lib, u, curve=curve, out=out, pts=pts, n=n, sc=sc) == (INVAL, DEV + OVERLAP), (curve, out - base)
            assert _host(lib, u, curve=curve, out=out, pts=pts, n=n, sc=sc) == (INVAL, HOST + OVERLAP)
        # in place over flagged host rows: the rows move, so it is not in place
        assert _host(lib, u, curve=curve, out=base, pts=base, n=n, ffi=ab + 8) == (INVAL, HOST + OVERLAP)
    assert u.unchanged()


def test_misaligned_device_scalars(lib):
    u = Bufs()
    for sbytes, nbits in ((8, 8), (16, 8), (32, 255)):
        msg = DEV + ": d_scalars must be aligned to min(scalar_bytes, 16) bytes"
        assert _dev(lib, u, sc=u.sc.ctypes.data + 4, sbytes=sbytes, nbits=nbits) == (INVAL, msg)
    assert u.unchanged()


def test_bad_host_stride(lib):
    u = Bufs()
    for curve, ab in ((0, 96), (1, 64), (3, 192)):
        for ffi in (8, ab - 4):
            assert _host(lib, u, curve=curve, ffi=ffi) == (INVAL, HOST + ": affine stride too small")
        for ffi in (ab + 1, ab + 2, ab + 9):
            assert _host(lib, u, curve=curve, ffi=ffi) == (INVAL, HOST + ": affine stride must be a multiple of 4 bytes")
    assert u.unchanged()


def test_well_formed_calls_reach_the_device_lookup(lib):
    """every refusal above comes before the device is looked for; a well-formed call (in place
    included) fails only for want of a device on a host without one"""
    if not _no_gpu():
        pytest.skip("a GPU is present; these calls fail only where there is no device")
    u = Bufs()
    base = u.out.ctypes.data
    for curve in range(8):
        for sbytes, nbits in ((4, 1), (8, 64), (16, 100), (32, 255)):
            assert _dev(lib, u, curve=curve, n=1, sbytes=sbytes, nbits=nbits)[0] == NODEV
            assert _host(lib, u, curve=curve, n=1, sbytes=sbytes, nbits=nbits)[0] == NODEV
        assert _dev(lib, u, curve=curve, out=base, pts=base, n=1)[0] == NODEV
        assert _host(lib, u, curve=curve, out=base, pts=base, n=1)[0] == NODEV
    assert _host(lib, u, curve=0, n=2, ffi=104)[0] == NODEV
    assert u.unchanged()


def test_python_argument_checks():
    from sppark_b200 import msm
    pts = np.zeros((3, 12), dtype=np.uint64)
    with pytest.raises(ValueError):
        msm.scale_points(msm.BLS12_381_G1, pts, np.zeros((2, 4), dtype=np.uint64))
    with pytest.raises(ValueError):
        msm.scale_points(msm.BLS12_381_G1, pts, np.zeros(3, dtype=np.uint32), nbits=33)
    with pytest.raises(TypeError):
        msm.scale_points(msm.BLS12_381_G1, pts, np.zeros((3, 3), dtype=np.uint64))
