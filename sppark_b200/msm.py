"""Host-side mirror of the reference's msm-cuda crate (poc/msm-cuda/src/lib.rs:18-81):
multi_scalar_mult (blst layout, 96-byte affine points) and multi_scalar_mult_arkworks
(arkworks layout, 104-byte G1Affine with an infinity flag), through the C-ABI.

Arrays: points (n, 12) uint64 [or (n, 13) for the arkworks layout: X, Y, flag word],
scalars (n, 4) uint64 little-endian, result (18,) uint64 = Jacobian {X, Y, Z} in Montgomery form.
"""
import numpy as np

from . import _lib

BLS12_381_G1, PALLAS, VESTA, BLS12_381_G2, BN254_G1, BLS12_377_G1, BN254_G2, BLS12_377_G2 = 0, 1, 2, 3, 4, 5, 6, 7
_LIMBS = {BLS12_381_G1: 6, PALLAS: 4, VESTA: 4, BLS12_381_G2: 12, BN254_G1: 4, BLS12_377_G1: 6, BN254_G2: 8, BLS12_377_G2: 12}    # 64-bit limbs per coordinate


def _check(points, scalars):
    if points.shape[0] != scalars.shape[0]:
        raise ValueError("length mismatch")                  # same panic as the crate (lib.rs:33-35)
    if not (points.flags["C_CONTIGUOUS"] and scalars.flags["C_CONTIGUOUS"]):
        raise TypeError("points and scalars must be C-contiguous")
    if points.dtype != np.uint64 or scalars.dtype != np.uint64 or scalars.shape[1] != 4:
        raise TypeError("points/scalars must be uint64 limb arrays")


def multi_scalar_mult(points, scalars):
    """blst_p1_affine[] x blst_scalar[] -> blst_p1  via mult_pippenger."""
    _check(points, scalars)
    assert points.shape[1] == 12
    out = np.zeros(18, dtype=np.uint64)
    err = _lib.lib().mult_pippenger(out.ctypes.data, points.ctypes.data, points.shape[0], scalars.ctypes.data)
    _lib.check(err)
    return out


def multi_scalar_mult_arkworks(points, scalars):
    """ark G1Affine[] (X, Y, infinity flag; size_of::<G1Affine>() == 104) x BigInteger256[]
    via mult_pippenger_inf."""
    _check(points, scalars)
    assert points.shape[1] == 13
    out = np.zeros(18, dtype=np.uint64)
    err = _lib.lib().mult_pippenger_inf(out.ctypes.data, points.ctypes.data, points.shape[0],
                                        scalars.ctypes.data, points.strides[0])
    _lib.check(err)
    return out


def multi_scalar_mult_fp2_arkworks(points, scalars):
    """ark G2Affine[] (X, Y in Fq2, infinity flag; size_of::<G2Affine>() == 200) x BigInteger256[]
    -> G2Projective (36 limbs) via mult_pippenger_fp2_inf (poc/msm-cuda/src/lib.rs:84-119)."""
    _check(points, scalars)
    assert points.shape[1] == 25
    out = np.zeros(36, dtype=np.uint64)
    err = _lib.lib().mult_pippenger_fp2_inf(out.ctypes.data, points.ctypes.data, points.shape[0],
                                            scalars.ctypes.data, points.strides[0])
    _lib.check(err)
    return out


def _scalar_bytes(scalars, u64, u32):
    """bytes per scalar from the array's shape and dtype: (n, 4) 64-bit words 32, (n, 2) 16, (n,) 64-bit 8,
    (n,) 32-bit 4; None for any other array"""
    if scalars.ndim == 2 and scalars.dtype == u64 and scalars.shape[1] in (2, 4):
        return 8 * scalars.shape[1]
    if scalars.ndim == 1 and scalars.dtype in (u64, u32):
        return 8 if scalars.dtype == u64 else 4
    return None


def _scalar_format(sbytes, mont, nbits):
    """(scalar_bytes, nbits) of a small-scalar call, or None for today's 32-byte call"""
    if sbytes == 32 and nbits is None:
        return None
    if mont:
        raise ValueError("mont=True takes (n, 4) scalars without nbits")
    if nbits is None:
        nbits = min(255, 8 * sbytes)
    if not 1 <= nbits <= min(255, 8 * sbytes):
        raise ValueError(f"nbits must be in [1, {min(255, 8 * sbytes)}] for {sbytes}-byte scalars")
    return sbytes, int(nbits)


def _host_format(scalars, mont, nbits):
    sbytes = _scalar_bytes(scalars, np.uint64, np.uint32)
    if sbytes is None:
        raise TypeError("scalars must be (n, 4) or (n, 2) uint64, (n,) uint64 or (n,) uint32")
    return _scalar_format(sbytes, mont, nbits)


def _check_compact(points, scalars):
    if points.shape[0] != scalars.shape[0]:
        raise ValueError("length mismatch")
    if not (points.flags["C_CONTIGUOUS"] and scalars.flags["C_CONTIGUOUS"]):
        raise TypeError("points and scalars must be C-contiguous")
    if points.dtype != np.uint64:
        raise TypeError("points must be a uint64 limb array")


def msm(curve, points, scalars, mont=False, nbits=None):
    """Any supported curve; host arrays of packed affine points (n, 2*limbs) or rows with an
    infinity-flag word appended (n, 2*limbs + 1).  mont=True: the scalars are Montgomery residues
    (the `mont` flag of the reference's C++ template, msm/pippenger.cuh:730-733).

    Small scalars: the scalar width follows the array, (n, 4) uint64 32 bytes, (n, 2) uint64 16,
    (n,) uint64 8, (n,) uint32 4; bits from `nbits` up are ignored (default min(255, 8 * width)).
    Fewer bits mean fewer windows and fewer bytes over PCIe (DESIGN.md section 5c)."""
    fmt = _host_format(scalars, mont, nbits)
    if fmt is None:
        _check(points, scalars)
    else:
        _check_compact(points, scalars)
    nl = _LIMBS[curve]
    assert points.shape[1] in (2 * nl, 2 * nl + 1)
    out = np.zeros(3 * nl, dtype=np.uint64)
    if fmt is None:
        err = _lib.lib().sppark_b200_msm_ex(curve, out.ctypes.data, points.ctypes.data, points.shape[0],
                                            scalars.ctypes.data, points.strides[0], int(mont))
    else:
        err = _lib.lib().sppark_b200_msm_bits(curve, out.ctypes.data, points.ctypes.data, points.shape[0],
                                              scalars.ctypes.data, points.strides[0], *fmt)
    _lib.check(err)
    return out


class MsmContext:
    """Points preloaded on the current GPU (the reference's msm_t{points, npoints}): every
    `invoke(scalars)` moves only the scalars.  Host arrays as for msm().

    precompute=K (an integer >= 1): store up to K shifted copies 2^(c*V*k) * P of the points, a
    fixed-base table that folds the scalar's D digits into V = ceil(D/K) bucket sets (DESIGN.md
    section 5a); it takes up to K times the device memory of the points."""

    def __init__(self, curve, points, precompute=None):
        import ctypes as C
        if points.dtype != np.uint64 or not points.flags["C_CONTIGUOUS"]:
            raise TypeError("points must be a C-contiguous uint64 limb array")
        nl = _LIMBS[curve]
        assert points.shape[1] in (2 * nl, 2 * nl + 1)
        self.curve, self.npoints, self._h = curve, points.shape[0], C.c_void_p()
        if precompute is None:
            err = _lib.lib().sppark_b200_msm_ctx_create(curve, points.ctypes.data, points.shape[0],
                                                        points.strides[0], C.byref(self._h))
        else:
            err = _lib.lib().sppark_b200_msm_ctx_create_precomputed(curve, points.ctypes.data, points.shape[0],
                                                                    points.strides[0], int(precompute),
                                                                    C.byref(self._h))
        _lib.check(err)

    def invoke(self, scalars, mont=False, nbits=None):
        """scalars: (n, 4) uint64, or a small-scalar array with an optional bit bound as for msm()"""
        fmt = _host_format(scalars, mont, nbits) if scalars.dtype in (np.uint64, np.uint32) else None
        if fmt is None and (scalars.dtype != np.uint64 or scalars.ndim != 2 or scalars.shape[1] != 4
                            or not scalars.flags["C_CONTIGUOUS"]):
            raise TypeError("scalars must be a C-contiguous (n, 4) uint64 array")
        if fmt is not None and not scalars.flags["C_CONTIGUOUS"]:
            raise TypeError("scalars must be C-contiguous")
        out = np.zeros(3 * _LIMBS[self.curve], dtype=np.uint64)
        if fmt is None:
            err = _lib.lib().sppark_b200_msm_ctx_invoke(self._h, out.ctypes.data, scalars.ctypes.data,
                                                        scalars.shape[0], int(mont))
        else:
            err = _lib.lib().sppark_b200_msm_ctx_invoke_bits(self._h, out.ctypes.data, scalars.ctypes.data,
                                                             scalars.shape[0], *fmt)
        _lib.check(err)
        return out

    def invoke_batch(self, scalars, nbits=None):
        """B scalar vectors against the preloaded points in one call: scalars (B, n, 4) or (B, n, 2)
        uint64, or (B, n) uint64 or uint32, the width following the array as for msm() (plain
        integers, bits from `nbits` up ignored).  Returns (B, 3 * limbs) uint64, row b the Jacobian
        result of vector b.  The vectors share the sort, accumulate, reduce and finish launches
        (DESIGN.md section 5d)."""
        sbytes, B, n = _batch_format(scalars, np.uint64, np.uint32)
        if not scalars.flags["C_CONTIGUOUS"]:
            raise TypeError("scalars must be C-contiguous")
        fmt = _scalar_format(sbytes, False, nbits) or (32, 255)
        out = np.zeros((B, 3 * _LIMBS[self.curve]), dtype=np.uint64)
        err = _lib.lib().sppark_b200_msm_ctx_invoke_batch(self._h, out.ctypes.data, scalars.ctypes.data, n, B, *fmt)
        _lib.check(err)
        return out

    def close(self):
        if self._h:
            _lib.lib().sppark_b200_msm_ctx_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def msm_dev(curve, d_points, d_scalars, npoints=None, stream=None, nbits=None):
    """msm_t::invoke with device-resident inputs (msm/pippenger.cuh:582-601): torch CUDA tensors
    of packed affine points / 32-byte scalars; synchronises the stream and returns the Jacobian
    result as a host array.

    Small scalars as for msm(), with int64 / int32 tensors: (n, 2) int64 16 bytes, (n,) int64 8,
    (n,) int32 4; bits from `nbits` up are ignored.  Any other tensor holds 32-byte scalars."""
    import torch
    nl = _LIMBS[curve]
    assert d_points.is_cuda and d_scalars.is_cuda and d_points.is_contiguous() and d_scalars.is_contiguous()
    sbytes = _scalar_bytes(d_scalars, torch.int64, torch.int32)
    if sbytes is None and nbits is not None:
        raise TypeError("a bit bound takes (n, 4) or (n, 2) int64, (n,) int64 or (n,) int32 scalars")
    fmt = _scalar_format(sbytes or 32, False, nbits)
    n = npoints if npoints is not None else d_scalars.numel() * d_scalars.element_size() // (fmt[0] if fmt else 32)
    out = np.zeros(3 * nl, dtype=np.uint64)
    with torch.cuda.device(d_points.device):
        s = stream if stream is not None else torch.cuda.current_stream().cuda_stream
        if fmt is None:
            err = _lib.lib().sppark_b200_msm_dev(curve, out.ctypes.data, d_points.data_ptr(), n,
                                                 d_scalars.data_ptr(), s)
        else:
            err = _lib.lib().sppark_b200_msm_dev_bits(curve, out.ctypes.data, d_points.data_ptr(), n,
                                                      d_scalars.data_ptr(), fmt[0], fmt[1], s)
    _lib.check(err)
    return out


def _batch_format(scalars, u64, u32):
    """(scalar_bytes, B, n) of a batch of B vectors of n scalars: (B, n, 4) / (B, n, 2) of 64-bit words,
    (B, n) of 64- or 32-bit scalars"""
    sbytes = None
    if scalars.ndim == 3 and scalars.dtype == u64 and scalars.shape[2] in (2, 4):
        sbytes = 8 * scalars.shape[2]
    elif scalars.ndim == 2 and scalars.dtype in (u64, u32):
        sbytes = 8 if scalars.dtype == u64 else 4
    if sbytes is None:
        raise TypeError("batched scalars must be (B, n, 4) or (B, n, 2) 64-bit words, or (B, n) of 64- or 32-bit "
                        "scalars")
    return sbytes, int(scalars.shape[0]), int(scalars.shape[1])


def msm_dev_batch(curve, d_points, d_scalars, nbits=None, stream=None):
    """B scalar vectors against one device point set in one call: torch CUDA tensors, d_points packed
    affine as for msm_dev, d_scalars (B, n, 4) or (B, n, 2) int64, or (B, n) int64 or int32 (the
    msm_dev conventions, plain integers, bits from `nbits` up ignored).  Synchronises the stream and
    returns (B, 3 * limbs) uint64, row b the Jacobian result of vector b."""
    import torch
    nl = _LIMBS[curve]
    assert d_points.is_cuda and d_scalars.is_cuda and d_points.is_contiguous() and d_scalars.is_contiguous()
    sbytes, B, n = _batch_format(d_scalars, torch.int64, torch.int32)
    fmt = _scalar_format(sbytes, False, nbits) or (32, 255)
    out = np.zeros((B, 3 * nl), dtype=np.uint64)
    with torch.cuda.device(d_points.device):
        s = stream if stream is not None else torch.cuda.current_stream().cuda_stream
        err = _lib.lib().sppark_b200_msm_dev_batch(curve, out.ctypes.data, d_points.data_ptr(), n,
                                                   d_scalars.data_ptr(), B, fmt[0], fmt[1], s)
    _lib.check(err)
    return out


def scale_points(curve, points, scalars, nbits=None):
    """out[i] = scalars[i] * points[i] on the GPU, host arrays: points packed affine (n, 2*limbs) uint64 or
    rows with an infinity-flag word appended (n, 2*limbs + 1); scalars as for msm() ((n, 4) or (n, 2)
    uint64, (n,) uint64 or uint32; plain integers, not reduced mod r, bits from `nbits` up ignored).
    Returns (n, 2*limbs) uint64 packed affine rows, infinity (0, 0) -- rows MsmContext and msm() take as
    they are.  Not constant-time (DESIGN.md section 5e)."""
    fmt = _host_format(scalars, False, nbits) or (32, 255)
    _check_compact(points, scalars)
    nl = _LIMBS[curve]
    assert points.ndim == 2 and points.shape[1] in (2 * nl, 2 * nl + 1)
    out = np.zeros((points.shape[0], 2 * nl), dtype=np.uint64)
    ffi = 0 if points.shape[1] == 2 * nl else points.strides[0]
    err = _lib.lib().sppark_b200_scale_points(curve, out.ctypes.data, points.ctypes.data, points.shape[0],
                                              scalars.ctypes.data, ffi, *fmt)
    _lib.check(err)
    return out


def scale_points_dev(curve, d_points, d_scalars, nbits=None, out=None, stream=None):
    """out[i] = d_scalars[i] * d_points[i] with torch CUDA tensors: d_points packed affine (n, 2*limbs)
    int64, d_scalars as for msm_dev ((n, 4) or (n, 2) int64, (n,) int64 or int32).  `out` (a tensor of
    d_points' shape, or d_points itself for in place) or a new tensor receives the packed affine rows.
    The work is enqueued on `stream` (default: the current stream) and not waited for."""
    import torch
    nl = _LIMBS[curve]
    assert d_points.is_cuda and d_scalars.is_cuda and d_points.is_contiguous() and d_scalars.is_contiguous()
    if d_points.ndim != 2 or d_points.shape[1] != 2 * nl:
        raise ValueError(f"d_points must be (n, {2 * nl}) packed affine rows")
    sbytes = _scalar_bytes(d_scalars, torch.int64, torch.int32)
    if sbytes is None:
        raise TypeError("scalars must be (n, 4) or (n, 2) int64, (n,) int64 or (n,) int32")
    fmt = _scalar_format(sbytes, False, nbits) or (32, 255)
    n = d_points.shape[0]
    if d_scalars.shape[0] != n:
        raise ValueError("length mismatch")
    if out is None:
        out = torch.empty_like(d_points)
    elif out.shape != d_points.shape or out.device != d_points.device or not out.is_contiguous():
        raise ValueError("out must be a contiguous tensor of d_points' shape on its device")
    with torch.cuda.device(d_points.device):
        s = stream if stream is not None else torch.cuda.current_stream().cuda_stream
        err = _lib.lib().sppark_b200_scale_points_dev(curve, out.data_ptr(), d_points.data_ptr(), n,
                                                      d_scalars.data_ptr(), fmt[0], fmt[1], s)
    _lib.check(err)
    return out


def generate_points_dev(curve, n, device=None):
    """(n, 2*limbs) int64 CUDA tensor holding (i+1)*G, i < n, as packed Montgomery affine points."""
    import torch
    nl = _LIMBS[curve]
    out = torch.empty((n, 2 * nl), dtype=torch.int64, device=device or "cuda")
    with torch.cuda.device(out.device):
        err = _lib.lib().sppark_b200_generate_points_dev(curve, out.data_ptr(), n,
                                                         torch.cuda.current_stream().cuda_stream)
    _lib.check(err)
    return out


def combine(curve, partials):
    """Sum of Jacobian points: partials (count, 3*limbs) uint64 host array."""
    partials = np.ascontiguousarray(partials, dtype=np.uint64)
    out = np.zeros(3 * _LIMBS[curve], dtype=np.uint64)
    _lib.check(_lib.lib().sppark_b200_msm_combine(curve, out.ctypes.data, partials.ctypes.data, partials.shape[0]))
    return out


def selftest_field(field, op, a, b):
    """Element-wise field op on the device, on Montgomery-form rows.  "msub4" takes a = (a_i, c_i)
    and b = (b_i, d_i) interleaved, 2n rows each, and returns the n rows a_i*b_i - c_i*d_i."""
    a = np.ascontiguousarray(a, dtype=np.uint64)
    b = np.ascontiguousarray(b, dtype=np.uint64)
    if a.shape != b.shape or (op == "msub4" and a.shape[0] % 2):
        raise ValueError("selftest_field: operand shapes")
    n = a.shape[0] // 2 if op == "msub4" else a.shape[0]
    r = np.zeros((n, a.shape[1]), dtype=np.uint64)
    ops = {"mul": 0, "add": 1, "sub": 2, "sqr": 3, "mul_shared": 4, "sqr_shared": 5, "msub_shared": 6, "msub4": 7}
    err = _lib.lib().sppark_b200_selftest_field(field, ops[op], n, r.ctypes.data, a.ctypes.data, b.ctypes.data)
    _lib.check(err)
    return r
