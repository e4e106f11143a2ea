"""The refusals of the MSM C entry points: for every entry, what a refused call returns -- the code and
the exact message --, whether the output was set to infinity (all-zero Jacobian points) or left as it
was, and whether the refusal comes before the device is looked for (-cudaErrorInvalidValue, -1, on any
host) or after it (-cudaErrorNoDevice, -100, on a host without a GPU).  No call here reads its point or
scalar buffers, so on a host with a GPU the refusals after the device lookup give their own code and
message.  The refusals that need a live context are at the end, marked gpu.
The scalar-multiplication entries are pinned in test_scale_points.py, the batch entries' codes in
test_msm_batch.py and the small-scalar codes in test_msm_small_scalars.py."""
import ctypes as C

import numpy as np
import pytest

INVAL, NODEV, BADDEV = -1, -100, -101
FILL = 0x5A
# per curve id (SPPARK_CURVE_*): packed affine {X, Y} and Jacobian {X, Y, Z} bytes
AFFINE = [96, 64, 64, 192, 64, 96, 128, 192]
JACOBIAN = [144, 96, 96, 288, 96, 144, 192, 288]
UNKNOWN = (8, 9, -1)
FORMAT = ": scalar_bytes must be 4, 8, 16 or 32 and 1 <= nbits <= min(255, 8 * scalar_bytes)"
ALIGN = ": d_scalars must be aligned to min(scalar_bytes, 16) bytes"
SMALL, MULT4 = "msm: affine stride too small", "msm: affine stride must be a multiple of 4 bytes"
NPOINTS = "msm: npoints must be < 2^31"
BIG = (1 << 31, (1 << 31) + 5, 1 << 40)


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
    """host buffers handed to the entries as points, scalars, device ids and output; the output is
    filled with FILL, so that a refusal shows whether it wrote infinity"""

    def __init__(self):
        self.pts = np.arange(1, 1 + 512, dtype=np.uint64)
        self.sc = np.arange(700, 700 + 512, dtype=np.uint64)
        self.ids = np.zeros(80, dtype=np.int32)
        self.out = np.full(4 * 288 + 64, FILL, dtype=np.uint8)
        self.ctx = C.c_void_p(0x1234)
        self.keep = [a.copy() for a in (self.pts, self.sc, self.ids)]

    @property
    def o(self):
        return self.out.ctypes.data

    @property
    def p(self):
        return self.pts.ctypes.data

    @property
    def s(self):
        return self.sc.ctypes.data

    def inputs_unchanged(self):
        return all(np.array_equal(a, b) for a, b in zip((self.pts, self.sc, self.ids), self.keep))

    def untouched(self):
        return self.inputs_unchanged() and (self.out == FILL).all()

    def infinity(self, nbytes):
        """the first nbytes of the output are zero, the rest as it was; refilled for the next call"""
        ok = self.inputs_unchanged() and not self.out[:nbytes].any() and (self.out[nbytes:] == FILL).all()
        self.out[:] = FILL
        return ok


def _host_entries(u):
    """the host-scalar MSM entries on one curve, as (name, curve, call(npoints, ffi_affine_sz))"""
    return [
        ("mult_pippenger_inf", 0, lambda n, f: ("mult_pippenger_inf", u.o, u.p, n, u.s, f)),
        ("mult_pippenger_fp2_inf", 3, lambda n, f: ("mult_pippenger_fp2_inf", u.o, u.p, n, u.s, f)),
        ("sppark_b200_msm", 0, lambda n, f: ("sppark_b200_msm", 0, u.o, u.p, n, u.s, f)),
        ("sppark_b200_msm", 1, lambda n, f: ("sppark_b200_msm", 1, u.o, u.p, n, u.s, f)),
        ("sppark_b200_msm_ex", 3, lambda n, f: ("sppark_b200_msm_ex", 3, u.o, u.p, n, u.s, f, 1)),
        ("sppark_b200_msm_bits", 0, lambda n, f: ("sppark_b200_msm_bits", 0, u.o, u.p, n, u.s, f, 8, 64)),
    ]


def _strides(name, curve):
    """(ffi_affine_sz, message) pairs of a bad host stride; the _inf entries always read the flag"""
    ab = AFFINE[curve]
    if name.startswith("mult_pippenger"):
        return [(0, SMALL), (8, SMALL), (ab, SMALL), (ab + 1, MULT4), (ab + 2, MULT4), (ab + 9, MULT4)]
    return [(8, SMALL), (ab - 4, SMALL), (ab + 1, MULT4), (ab + 2, MULT4), (ab + 9, MULT4)]


def _after_device(got, msg):
    """a refusal after the device lookup: its own code and message where there is a GPU"""
    if _no_gpu():
        return got[0] == NODEV
    return got == (INVAL, msg)


# ---- refusals before the device lookup ------------------------------------------------------------
UNKNOWN_CURVE_MSG = {
    "sppark_b200_msm": "sppark_b200_msm: unknown curve",
    "sppark_b200_msm_ex": "sppark_b200_msm: unknown curve",
    "sppark_b200_msm_bits": "sppark_b200_msm_bits: unknown curve",
    "sppark_b200_msm_dev": "sppark_b200_msm_dev: unknown curve",
    "sppark_b200_msm_dev_bits": "sppark_b200_msm_dev_bits: unknown curve",
    "sppark_b200_msm_dev_batch": "sppark_b200_msm_dev_batch: unknown curve",
    "sppark_b200_msm_ctx_create": "msm_ctx_create: unknown curve",
    "sppark_b200_msm_ctx_create_precomputed": "msm_ctx_create: unknown curve",
    "sppark_b200_msm_sharded": "msm_sharded: unknown curve",
    "sppark_b200_msm_combine": "msm_combine: unknown curve",
    "sppark_b200_generate_points_dev": "generate_points: unknown curve",
}


def _curve_call(u, name, c):
    return {
        "sppark_b200_msm": (c, u.o, u.p, 4, u.s, 0),
        "sppark_b200_msm_ex": (c, u.o, u.p, 4, u.s, 0, 1),
        "sppark_b200_msm_bits": (c, u.o, u.p, 4, u.s, 0, 3, 8),                 # the curve before the format
        "sppark_b200_msm_dev": (c, u.o, u.p, 4, u.s, None),
        "sppark_b200_msm_dev_bits": (c, u.o, u.p, 4, u.s + 4, 3, 8, None),
        "sppark_b200_msm_dev_batch": (c, u.o, u.p, 4, u.s, 2, 32, 255, None),
        "sppark_b200_msm_ctx_create": (c, u.p, 4, 8, C.byref(u.ctx)),           # and before the stride
        "sppark_b200_msm_ctx_create_precomputed": (c, u.p, 4, 0, 2, C.byref(u.ctx)),
        "sppark_b200_msm_sharded": (c, None, u.p, 4, u.s, 0, 0, None, 0),       # and before the output
        "sppark_b200_msm_combine": (c, u.o, u.s, 2),
        "sppark_b200_generate_points_dev": (c, u.o, 4, None),
    }[name]


@pytest.mark.parametrize("name", sorted(UNKNOWN_CURVE_MSG))
def test_unknown_curve(lib, name):
    u = Bufs()
    for c in UNKNOWN:
        assert _call(lib, name, *_curve_call(u, name, c)) == (INVAL, UNKNOWN_CURVE_MSG[name]), c
        assert u.untouched()
    if "ctx_create" in name:
        assert u.ctx.value is None                       # *out is cleared before the curve is looked up


def test_bad_scalar_format_and_alignment_messages(lib):
    """the messages of the format and alignment refusals; test_msm_small_scalars pins their codes"""
    u = Bufs()
    for sb, nb in ((3, 8), (4, 33), (32, 256)):
        got = _call(lib, "sppark_b200_msm_bits", 1, u.o, u.p, 4, u.s, 0, sb, nb)
        assert got == (INVAL, "sppark_b200_msm_bits" + FORMAT) and u.infinity(JACOBIAN[1])
        got = _call(lib, "sppark_b200_msm_dev_bits", 3, u.o, u.p, 4, u.s, sb, nb, None)
        assert got == (INVAL, "sppark_b200_msm_dev_bits" + FORMAT) and u.infinity(JACOBIAN[3])
        got = _call(lib, "sppark_b200_msm_dev_batch", 0, u.o, u.p, 4, u.s, 3, sb, nb, None)
        assert got == (INVAL, "sppark_b200_msm_dev_batch" + FORMAT) and u.infinity(3 * JACOBIAN[0])
    for sb in (8, 16, 32):
        got = _call(lib, "sppark_b200_msm_dev_bits", 0, u.o, u.p, 4, u.s + 4, sb, 8, None)
        assert got == (INVAL, "sppark_b200_msm_dev_bits" + ALIGN) and u.infinity(JACOBIAN[0])
        got = _call(lib, "sppark_b200_msm_dev_batch", 1, u.o, u.p, 4, u.s + 4, 2, sb, 8, None)
        assert got == (INVAL, "sppark_b200_msm_dev_batch" + ALIGN) and u.infinity(2 * JACOBIAN[1])
    assert u.untouched()


def test_null_context(lib):
    u = Bufs()
    for n in (0, 4):
        assert (_call(lib, "sppark_b200_msm_ctx_invoke", None, u.o, u.s, n, 0)
                == (INVAL, "msm_ctx_invoke: more scalars than preloaded points"))
        # the context is checked before the format
        for sb, nb in ((32, 255), (3, 8)):
            assert (_call(lib, "sppark_b200_msm_ctx_invoke_bits", None, u.o, u.s, n, sb, nb)
                    == (INVAL, "msm_ctx_invoke_bits: null context"))
        assert (_call(lib, "sppark_b200_msm_ctx_invoke_batch", None, u.o, u.s, n, 2, 32, 255)
                == (INVAL, "msm_ctx_invoke_batch: null context"))
    assert u.untouched()


def test_ctx_create_null_output_and_copies(lib):
    u = Bufs()
    for c in (0, 3) + UNKNOWN:
        assert (_call(lib, "sppark_b200_msm_ctx_create", c, u.p, 4, 0, None)
                == (INVAL, "msm_ctx_create: null output"))
        assert (_call(lib, "sppark_b200_msm_ctx_create_precomputed", c, u.p, 4, 0, 2, None)
                == (INVAL, "msm_ctx_create: null output"))
        # copies == 0 before the output and the curve
        for out in (None, C.byref(u.ctx)):
            assert (_call(lib, "sppark_b200_msm_ctx_create_precomputed", c, u.p, 4, 8, 0, out)
                    == (INVAL, "msm_ctx_create_precomputed: copies must be >= 1"))
        assert u.ctx.value is None
        u.ctx.value = 0x1234
    assert u.untouched()


def test_sharded_device_ids(lib):
    u = Bufs()
    ids = u.ids.ctypes.data
    msg = "msm_sharded: need 1..64 device ids"
    assert _call(lib, "sppark_b200_msm_sharded", 0, None, u.p, 4, u.s, 0, 0, ids, 1) == (INVAL, msg)
    assert u.untouched()
    for curve in (0, 1, 3):
        for args in ((ids, 0), (ids, 65), (None, 1), (None, 0)):
            assert _call(lib, "sppark_b200_msm_sharded", curve, u.o, u.p, 4, u.s, 0, 0, *args) == (INVAL, msg)
            assert u.infinity(JACOBIAN[curve])


def test_generate_points_size_before_curve(lib):
    u = Bufs()
    for c in (0, 3) + UNKNOWN:
        for n in BIG:
            assert _call(lib, "sppark_b200_generate_points_dev", c, u.o, n, None) == (INVAL, "generate_points: n too large")
    assert u.untouched()


def test_selftest_arguments(lib):
    u = Bufs()
    for f in (8, 9, -1):
        assert _call(lib, "sppark_b200_selftest_field", f, 0, 4, u.o, u.p, u.s) == (INVAL, "selftest: unknown field")
    info = np.zeros(5, dtype=np.uint32)
    a = [u.o] * 4 + [info.ctypes.data]
    for n, wbits, cap in ((0, 8, 0), (1 << 31, 8, 0), (64, 2, 0), (64, 25, 0), (64, 8, 24577)):
        assert (_call(lib, "sppark_b200_selftest_msm_sort", n, wbits, cap, u.s, *a)
                == (INVAL, "selftest_msm_sort: bad arguments"))
    assert u.untouched() and not info.any()


# ---- host stride and sizes of the host-point entries: before the device lookup ----------------------
def test_host_msm_bad_stride(lib):
    u = Bufs()
    for name, curve, call in _host_entries(u):
        for ffi, msg in _strides(name, curve):
            assert _call(lib, *call(4, ffi)) == (INVAL, msg), (name, curve, ffi)
            assert u.infinity(JACOBIAN[curve])


def test_host_msm_too_many_points(lib):
    u = Bufs()
    entries = _host_entries(u) + [("mult_pippenger", 0, lambda n, f: ("mult_pippenger", u.o, u.p, n, u.s))]
    for name, curve, call in entries:
        good = AFFINE[curve] + 8 if name.startswith("mult_pippenger") else 0
        for n in BIG:
            # the size before the stride
            for ffi in (good, 8):
                assert _call(lib, *call(n, ffi)) == (INVAL, NPOINTS), (name, n, ffi)
                assert u.infinity(JACOBIAN[curve])


def test_host_msm_no_points_ignores_the_stride(lib):
    """npoints == 0 is a no-op that writes infinity, after the device lookup"""
    u = Bufs()
    for name, curve, call in _host_entries(u):
        for ffi, _ in _strides(name, curve):
            code, _ = _call(lib, *call(0, ffi))
            assert code == (NODEV if _no_gpu() else 0), (name, ffi)
            assert u.infinity(JACOBIAN[curve])


def test_dev_msm_too_many_points(lib):
    """the device entries check the size after the device lookup"""
    u = Bufs()
    for n in BIG:
        assert _after_device(_call(lib, "sppark_b200_msm_dev", 0, u.o, u.p, n, u.s, None), NPOINTS)
        assert u.infinity(JACOBIAN[0])
        assert _after_device(_call(lib, "sppark_b200_msm_dev_bits", 3, u.o, u.p, n, u.s, 8, 64, None), NPOINTS)
        assert u.infinity(JACOBIAN[3])


def test_ctx_create_bad_stride_and_size(lib):
    u = Bufs()
    copies_msg = "msm: copies * npoints must be < 2^31"
    for curve in (0, 1, 3):
        ab = AFFINE[curve]
        # (npoints, ffi_affine_sz, message) of both entries
        for n, ffi, msg in [(4, 8, SMALL), (0, 8, SMALL), (4, ab - 4, SMALL), (4, ab + 1, MULT4), (4, ab + 2, MULT4),
                            (1 << 31, 8, SMALL),                    # the stride before the size
                            (1 << 31, 0, NPOINTS), (1 << 40, ab + 8, NPOINTS)]:
            for call in (("sppark_b200_msm_ctx_create", curve, u.p, n, ffi, C.byref(u.ctx)),
                         ("sppark_b200_msm_ctx_create_precomputed", curve, u.p, n, ffi, 3, C.byref(u.ctx))):
                assert _call(lib, *call) == (INVAL, msg), (curve, n, ffi)
                assert u.ctx.value is None
                u.ctx.value = 0x1234
        for n, ffi, copies in [(1 << 30, 0, 2), ((1 << 29) + 1, ab + 8, 4), (1 << 20, 0, 1 << 11),
                               (1, 0, 1 << 31)]:
            got = _call(lib, "sppark_b200_msm_ctx_create_precomputed", curve, u.p, n, ffi, copies, C.byref(u.ctx))
            assert got == (INVAL, copies_msg), (curve, n, copies)
            assert u.ctx.value is None
            u.ctx.value = 0x1234
    assert u.untouched()


def test_sharded_bad_device_id(lib):
    u = Bufs()
    for bad in (-1, 64, 1 << 20):
        u.ids[:] = 0
        u.ids[2] = bad
        u.keep[2] = u.ids.copy()
        got = _call(lib, "sppark_b200_msm_sharded", 0, u.o, u.p, 8, u.s, 0, 0, u.ids.ctypes.data, 3)
        if _no_gpu():
            assert got == (NODEV, "msm_sharded: no CUDA device")
        else:
            assert got == (BADDEV, "msm_sharded: no such device")
        assert u.infinity(JACOBIAN[0])


def test_sharded_bad_stride_and_chunk_size(lib):
    u = Bufs()
    ids = u.ids.ctypes.data
    for curve in (0, 1, 3):
        for ffi, msg in _strides("sppark_b200_msm", curve):
            got = _call(lib, "sppark_b200_msm_sharded", curve, u.o, u.p, 8, u.s, ffi, 0, ids, 2)
            assert got == (INVAL, msg)
            assert u.infinity(JACOBIAN[curve])
        for n, ndev in ((1 << 31, 1), (1 << 32, 2), (1 << 40, 3)):          # chunks of 2^31 points or more
            got = _call(lib, "sppark_b200_msm_sharded", curve, u.o, u.p, n, u.s, 0, 0, ids, ndev)
            assert got == (INVAL, NPOINTS)
            assert u.infinity(JACOBIAN[curve])


# ---- well-formed calls fail only for want of a device ---------------------------------------------
def test_well_formed_calls_reach_the_device_lookup(lib):
    if not _no_gpu():
        pytest.skip("a GPU is present; these calls fail only where there is no device")
    u = Bufs()
    ids = u.ids.ctypes.data
    jacobian_calls = [
        (0, ("mult_pippenger", u.o, u.p, 4, u.s)),
        (0, ("mult_pippenger_inf", u.o, u.p, 4, u.s, 104)),
        (3, ("mult_pippenger_fp2_inf", u.o, u.p, 4, u.s, 200)),
        (0, ("sppark_b200_msm_dev", 0, u.o, u.p, 4, u.s, None)),
        (1, ("sppark_b200_msm_dev_bits", 1, u.o, u.p, 4, u.s, 4, 32, None)),
    ]
    for curve in range(8):
        jacobian_calls += [(curve, ("sppark_b200_msm", curve, u.o, u.p, 4, u.s, 0)),
                           (curve, ("sppark_b200_msm_ex", curve, u.o, u.p, 0, u.s, 0, 1)),
                           (curve, ("sppark_b200_msm_bits", curve, u.o, u.p, 4, u.s, 0, 16, 100))]
    for curve, call in jacobian_calls:
        code, _ = _call(lib, *call)
        assert code == NODEV, call
        assert u.infinity(JACOBIAN[curve]), call
    for curve in range(8):
        for create in (("sppark_b200_msm_ctx_create", curve, u.p, 4, 0, C.byref(u.ctx)),
                       ("sppark_b200_msm_ctx_create_precomputed", curve, u.p, 4, 0, 3, C.byref(u.ctx))):
            assert _call(lib, *create)[0] == NODEV
            assert u.ctx.value is None
            u.ctx.value = 0x1234
        assert _call(lib, "sppark_b200_msm_combine", curve, u.o, u.s, 2)[0] == NODEV
        assert u.infinity(JACOBIAN[curve])
    # the 2^31 limit of a sharded MSM is per chunk: three chunks below it pass the checks
    for n in (8, (1 << 31) + 5, 3 * ((1 << 31) - 1)):
        got = _call(lib, "sppark_b200_msm_sharded", 0, u.o, u.p, n, u.s, 0, 0, ids, 3)
        assert got == (NODEV, "msm_sharded: no CUDA device")
        assert u.infinity(JACOBIAN[0])
    assert _call(lib, "sppark_b200_selftest_field", 0, 0, 4, u.o, u.p, u.s)[0] == NODEV
    info = np.zeros(5, dtype=np.uint32)
    assert _call(lib, "sppark_b200_selftest_msm_sort", 64, 8, 0, u.s, u.o, u.o, u.o, u.o, info.ctypes.data)[0] == NODEV
    assert u.untouched()


# ---- refusals of a live context ---------------------------------------------------------------------
def _ctx(lib, u, curve=0, n=4):
    rows = np.zeros(n * AFFINE[curve], dtype=np.uint8)             # points at infinity
    assert _call(lib, "sppark_b200_msm_ctx_create", curve, rows.ctypes.data, n, 0, C.byref(u.ctx)) == (0, None)
    return u.ctx.value


@pytest.mark.gpu
def test_ctx_more_scalars_than_points(lib):
    if _no_gpu():
        pytest.skip("needs a GPU")
    u = Bufs()
    for curve in (0, 3):
        ctx = _ctx(lib, u, curve)
        try:
            got = _call(lib, "sppark_b200_msm_ctx_invoke", ctx, u.o, u.s, 5, 0)
            assert got == (INVAL, "msm_ctx_invoke: more scalars than preloaded points")
            assert u.infinity(JACOBIAN[curve])
            got = _call(lib, "sppark_b200_msm_ctx_invoke_bits", ctx, u.o, u.s, 5, 8, 64)
            assert got == (INVAL, "msm_ctx_invoke_bits: more scalars than preloaded points")
            assert u.infinity(JACOBIAN[curve])
            got = _call(lib, "sppark_b200_msm_ctx_invoke_bits", ctx, u.o, u.s, 5, 8, 65)   # the format first
            assert got == (INVAL, "msm_ctx_invoke_bits" + FORMAT) and u.infinity(JACOBIAN[curve])
            got = _call(lib, "sppark_b200_msm_ctx_invoke_batch", ctx, u.o, u.s, 5, 3, 8, 64)
            assert got == (INVAL, "msm_ctx_invoke_batch: more scalars than preloaded points")
            assert u.infinity(3 * JACOBIAN[curve])
        finally:
            lib.sppark_b200_msm_ctx_free(ctx)


@pytest.mark.gpu
def test_ctx_on_another_device(lib):
    if _no_gpu() or lib.sppark_b200_ngpus() < 2:
        pytest.skip("needs two GPUs")
    u = Bufs()
    assert lib.sppark_b200_sm_count(1) > 0                         # makes device 1 current
    ctx = _ctx(lib, u)
    try:
        assert lib.sppark_b200_sm_count(0) > 0
        got = _call(lib, "sppark_b200_msm_ctx_invoke", ctx, u.o, u.s, 4, 0)
        assert got == (BADDEV, "msm_ctx_invoke: the points live on another device")
        assert u.infinity(JACOBIAN[0])
        got = _call(lib, "sppark_b200_msm_ctx_invoke_bits", ctx, u.o, u.s, 4, 8, 64)
        assert got == (BADDEV, "msm_ctx_invoke_bits: the points live on another device")
        assert u.infinity(JACOBIAN[0])
        got = _call(lib, "sppark_b200_msm_ctx_invoke_batch", ctx, u.o, u.s, 4, 2, 8, 64)
        assert got == (BADDEV, "msm_ctx_invoke_batch: the points live on another device")
        assert u.infinity(2 * JACOBIAN[0])
    finally:
        lib.sppark_b200_msm_ctx_free(ctx)
