"""Batched MSM on the CPU: the CPU single-stepper tests/emu/msm_batch_emu.cpp runs the batched bin sort,
accumulate, reduce and finish (csrc/msm/msm_core.cuh with Config::nvecs > 1) over groups of vectors,
and every vector's result is compared with the oracle; then the argument checks of the two batch
entries of the C ABI, without a device."""
import ctypes as C
import random

import numpy as np
import pytest

from test_emu import R_BLS, _build

P_ORDER = None       # Pallas' group order: Vesta's base field, read from the oracle


@pytest.fixture(scope="module")
def emu():
    l = _build("msm_batch_emu")
    for fn in (l.emu_batch_bls12_381, l.emu_batch_pallas):
        fn.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_size_t] + [C.c_uint] * 8 + \
                      [C.c_void_p]
    return l


@pytest.fixture
def clean_env(monkeypatch):
    for k in ("SPPARK_B200_MSM_WBITS", "SPPARK_B200_MSM_HEAVY"):
        monkeypatch.delenv(k, raising=False)
    return monkeypatch


def _pack(vals, sbytes):
    return np.frombuffer(b"".join(v.to_bytes(sbytes, "little") for v in vals), dtype=np.uint8).copy()


def _rows(vals):
    return np.array([[(v >> (64 * i)) & (2**64 - 1) for i in range(4)] for v in vals], dtype=np.uint64).reshape(-1, 4)


def _points(oracle, curve, N):
    base = oracle.gen_points(curve, 29)
    pts = base[np.arange(N) % 29].copy()
    if N > 3:
        pts[3] = 0
    return pts


def _run(oracle, emu, curve, pts, vecs, n, sbytes=32, nbits=255, wbits=0, copies=0, heavy=0, cap=0, wpg=0, group=0):
    """vecs: B lists of n integers (bits above nbits allowed); every result against the oracle"""
    nl = 6 if curve == "bls12_381" else 4
    B = len(vecs)
    sc = _pack([v for vec in vecs for v in vec], sbytes) if n else np.zeros(8, dtype=np.uint8)
    out, info = np.zeros((max(B, 1), 3 * nl), dtype=np.uint64), np.zeros(8, dtype=np.uint32)
    fn = emu.emu_batch_bls12_381 if curve == "bls12_381" else emu.emu_batch_pallas
    fn(out.ctypes.data, pts.ctypes.data, pts.shape[0], sc.ctypes.data, n, B, group, sbytes, nbits, wbits, copies,
       heavy, cap, wpg, info.ctypes.data)
    for b, vec in enumerate(vecs):
        want = oracle.msm(curve, pts[:n], _rows([v % (1 << nbits) for v in vec]), "pippenger", ncpus=4) if n else \
            np.zeros(3 * nl, dtype=np.uint64)
        got = oracle.jac_to_affine(curve, out[b]) if out[b].any() else None
        exp = oracle.jac_to_affine(curve, want) if want.any() else None
        assert (got is None and exp is None) or np.array_equal(got, exp), (curve, b, n, sbytes, nbits, wbits, copies)
    return [int(v) for v in info]


def _vecs(rnd, B, n, bound):
    return [[rnd.randrange(bound) for _ in range(n)] for _ in range(B)]


@pytest.mark.parametrize("B", [1, 2, 3, 4, 5])
@pytest.mark.parametrize("n", [1, 7, 40])
def test_batch_small(oracle, emu, clean_env, B, n):
    rnd = random.Random(B * 100 + n)
    pts = _points(oracle, "bls12_381", n)
    info = _run(oracle, emu, "bls12_381", pts, _vecs(rnd, B, n, R_BLS), n)
    assert info[5] == 1


@pytest.mark.parametrize("wbits", [3, 4, 5, 8, 13])
def test_batch_forced_widths(oracle, emu, clean_env, wbits):
    """every set of a vector is full-width except its thin top window: window groups of 3 sets in the
    bin histogram cross vector boundaries"""
    rnd = random.Random(wbits)
    n = 60
    pts = _points(oracle, "bls12_381", n)
    info = _run(oracle, emu, "bls12_381", pts, _vecs(rnd, 4, n, R_BLS), n, wbits=wbits, wpg=3)
    assert info[0] == wbits and info[1] == -(-256 // wbits)


@pytest.mark.parametrize("curve", ["bls12_381", "pallas"])
@pytest.mark.parametrize("K,wbits", [(2, 8), (4, 8), (4, 5), (2, 13)])
def test_batch_over_tables(oracle, emu, clean_env, curve, K, wbits):
    """a plain context and tables of K copies; the batch invokes a prefix of the preloaded points"""
    r = R_BLS if curve == "bls12_381" else oracle.ff_consts("vesta_fp")["p"]
    rnd = random.Random(K * 31 + wbits)
    N, n = 70, 53
    pts = _points(oracle, curve, N)
    vecs = _vecs(rnd, 3, n, r)
    info = _run(oracle, emu, curve, pts, vecs, n, wbits=wbits, copies=K, wpg=2)
    D = -(-256 // wbits)
    assert info[1] == -(-D // K) and info[3] == -(-D // info[1]), info
    _run(oracle, emu, curve, pts, vecs, n, wbits=wbits, copies=1)


@pytest.mark.parametrize("sbytes,nbits,wbits,copies", [(4, 1, 0, 0), (4, 16, 5, 0), (4, 32, 8, 0), (8, 33, 11, 0),
                                                       (8, 64, 0, 0), (16, 100, 10, 0), (16, 128, 7, 0),
                                                       (32, 200, 12, 0), (32, 255, 5, 0), (8, 64, 8, 4),
                                                       (16, 128, 13, 2), (4, 8, 8, 4)])
def test_batch_scalar_formats(oracle, emu, clean_env, sbytes, nbits, wbits, copies):
    """random bits above nbits are ignored in every vector"""
    rnd = random.Random(sbytes * 1000 + nbits)
    n = 45
    pts = _points(oracle, "bls12_381", n)
    _run(oracle, emu, "bls12_381", pts, _vecs(rnd, 3, n, 1 << (8 * sbytes)), n, sbytes, nbits, wbits, copies, wpg=4)


@pytest.mark.parametrize("group", [1, 2, 3])
@pytest.mark.parametrize("cap", [0, 8])
def test_batch_heavy_vector_next_to_zero_and_uniform(oracle, emu, clean_env, group, cap):
    """vector 0 uniform, vector 1 all zero, vector 2 one value everywhere (heavy buckets in that vector
    only), vector 3 uniform; groups of 1, 2 and all; a bin cap of 8 sends bins down the overflow path"""
    rnd = random.Random(group)
    n = 300
    pts = _points(oracle, "bls12_381", n)
    vecs = [_vecs(rnd, 1, n, R_BLS)[0], [0] * n, [R_BLS - 1] * n, _vecs(rnd, 1, n, R_BLS)[0]]
    info = _run(oracle, emu, "bls12_381", pts, vecs, n, wbits=7, heavy=20, cap=cap, group=group)
    assert info[5] == -(-4 // group)
    assert info[6] > 0 and (cap == 0) == (info[7] == 0), info


@pytest.mark.parametrize("group", [1, 2, 5])
def test_batch_group_splits(oracle, emu, clean_env, group):
    """five vectors in groups of 1, 2 (a short last group) and all five"""
    rnd = random.Random(77)
    n = 33
    pts = _points(oracle, "pallas", n)
    info = _run(oracle, emu, "pallas", pts, _vecs(rnd, 5, n, oracle.ff_consts("vesta_fp")["p"]), n, group=group)
    assert info[5] == -(-5 // group)


def test_batch_no_points(oracle, emu, clean_env):
    pts = _points(oracle, "bls12_381", 4)
    _run(oracle, emu, "bls12_381", pts, [[], [], []], 0)


# ---- C ABI: argument checks before any device work --------------------------------------------------
INVALID = -1


def _drop(lib, err):
    if err.message:
        lib.drop_error_message(err.message)
    return err.code


def _dev(lib, out, sbytes=8, nbits=64, batch=3, n=4, ptr=0x10000, curve=0):
    return _drop(lib, lib.sppark_b200_msm_dev_batch(curve, out.ctypes.data, ptr, n, ptr, batch, sbytes, nbits, None))


@pytest.mark.parametrize("sbytes,nbits", [(3, 8), (12, 8), (64, 8), (4, 0), (4, 33), (16, 129), (32, 256)])
def test_batch_bad_format_refused(lib, sbytes, nbits):
    out = np.ones((3, 18), dtype=np.uint64)
    assert _dev(lib, out, sbytes, nbits) == INVALID
    assert not out.any()


def test_batch_size_overflow_refused(lib):
    out = np.ones((3, 18), dtype=np.uint64)
    assert _dev(lib, out, 32, 255, batch=3, n=(1 << 62)) == INVALID
    assert not out.any()
    out = np.ones(18, dtype=np.uint64)
    assert _dev(lib, out, 32, 255, batch=1 << 62, n=1) == INVALID       # no output of that size exists: none written
    assert out.all()


def test_batch_misaligned_device_scalars_refused(lib):
    for sbytes in (8, 16, 32):
        out = np.ones((3, 18), dtype=np.uint64)
        assert _dev(lib, out, sbytes, 8, ptr=0x10004) == INVALID
        assert not out.any()


def test_batch_unknown_curve_and_null_context_refused(lib):
    out = np.ones((3, 18), dtype=np.uint64)
    assert _dev(lib, out, curve=8) == INVALID
    assert _dev(lib, out, curve=-1) == INVALID
    sc = np.zeros(96, dtype=np.uint8)
    assert _drop(lib, lib.sppark_b200_msm_ctx_invoke_batch(None, out.ctypes.data, sc.ctypes.data, 4, 3, 8, 64)) == INVALID
    assert out.all()                                     # the output size is unknown: nothing is written


def test_batch_of_zero_vectors_is_a_no_op(lib):
    out = np.ones(18, dtype=np.uint64)
    assert _dev(lib, out, batch=0) == 0
    assert out.all()


def test_python_batch_formats():
    from sppark_b200 import msm
    u64, u32 = np.uint64, np.uint32
    assert msm._batch_format(np.zeros((2, 3, 4), u64), u64, u32) == (32, 2, 3)
    assert msm._batch_format(np.zeros((2, 3, 2), u64), u64, u32) == (16, 2, 3)
    assert msm._batch_format(np.zeros((5, 3), u64), u64, u32) == (8, 5, 3)
    assert msm._batch_format(np.zeros((5, 3), u32), u64, u32) == (4, 5, 3)
    for bad in (np.zeros((2, 3, 3), u64), np.zeros(3, u64), np.zeros((2, 3), np.int16)):
        with pytest.raises(TypeError):
            msm._batch_format(bad, u64, u32)
