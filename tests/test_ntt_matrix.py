"""NTT and LDE down the columns of a row-major matrix, without a GPU: the matrix pass descriptors
(make_plan with one transform column per tile + set_matrix) run through the HD phase functions of
ntt_core.cuh by the CPU single-stepper tests/emu/ntt_matrix_emu.cpp, tile by tile over (transform
tile, column block); every column must equal the oracle's transform of that column.  Also: the
matrix C entry points and Python wrappers fail cleanly on a CPU-only host."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

EMU_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu", "ntt_matrix_emu.cpp")
GL_P = 2**64 - 2**32 + 1
BB_P = 0x78000001
NN, NR, RN, RR, BB = range(5)
WIDTHS = [1, 2, 3, 4, 5, 7, 8, 9, 16, 17, 33]
ALL = [(o, i, c) for o in range(5) for i in (0, 1) for c in (0, 1)]
SOME = [(NN, 0, 0), (NR, 1, 0), (RN, 0, 1), (RR, 1, 1), (BB, 0, 0), (BB, 1, 1)]


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("ntt_matrix_emu") / "libntt_matrix_emu.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-x", "c++", "-o", so, EMU_SRC])
    l = C.CDLL(so)
    l.emu_ntt_matrix.argtypes = [C.c_int, C.c_void_p, C.c_uint, C.c_uint64, C.c_int, C.c_int, C.c_int, C.c_uint]
    l.emu_lde_matrix.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_uint, C.c_uint, C.c_uint64, C.c_uint]
    l.emu_matrix_shape.argtypes = [C.c_uint, C.c_uint64, C.c_int, C.c_uint, C.c_uint]
    return l


def _brev_idx(lg):
    return np.array([int(format(i, f"0{lg}b")[::-1], 2) for i in range(1 << lg)]) if lg else np.zeros(1, int)


def _oracle_col(ofn, x, lg, order, inv, coset):
    """oracle transform of one column; the oracle has no coset BB, which is bitrev(coset NN(bitrev x))"""
    if coset and order == BB:
        idx = _brev_idx(lg)
        return ofn(x[idx], NN, bool(inv), True)[idx]
    return ofn(x, order, bool(inv), bool(coset))


def _matrix(field, lg, width, seed):
    rng = np.random.default_rng(seed)
    if field == 0:
        return rng.integers(0, GL_P, size=(1 << lg, width), dtype=np.uint64)
    return rng.integers(0, BB_P, size=(1 << lg, width), dtype=np.uint32)


def _check(oracle, emu, field, x, lg, lg_tile, combos=ALL, reduced=None):
    """x: (2^lg, width); reduced: what the oracle sees (x mod p for loose Goldilocks words)"""
    ofn = oracle.ntt_gl64 if field == 0 else oracle.ntt_bb31
    ref = x if reduced is None else reduced
    width = x.shape[1]
    for order, inv, coset in combos:
        y = x.copy()
        assert emu.emu_ntt_matrix(field, y.ctypes.data, lg, width, order, inv, coset, lg_tile) >= 1
        for c in range(width):
            want = _oracle_col(ofn, np.ascontiguousarray(ref[:, c]), lg, order, inv, coset)
            assert np.array_equal(y[:, c], want), (field, lg, width, lg_tile, order, inv, coset, c)


@pytest.mark.parametrize("lg", range(1, 15))
@pytest.mark.parametrize("field", [0, 1])
def test_matrix_columns_match_oracle(oracle, emu, field, lg, monkeypatch):
    """every lg of 1..14, all orders, directions and types; 2^7-element tiles from 2^5 on, so that
    the columns span several tiles and column blocks"""
    monkeypatch.delenv("SPPARK_B200_NTT_SPLIT", raising=False)
    width = WIDTHS[lg % len(WIDTHS)]
    while width > 1 and (width << lg) > 1 << 15:
        width = WIDTHS[WIDTHS.index(width) - 1]
    _check(oracle, emu, field, _matrix(field, lg, width, 100 * field + lg), lg, 7 if lg > 4 else 14)


@pytest.mark.parametrize("width", WIDTHS)
def test_matrix_widths(oracle, emu, width, monkeypatch):
    """widths below, at and straddling the column block: blocks of 4 (2^6 rows in 2^8-element
    tiles), of 32 (2^11-element tiles) and of 2 (a 2^9-row pass in 2^10-element tiles)"""
    monkeypatch.delenv("SPPARK_B200_NTT_SPLIT", raising=False)
    for field in (0, 1):
        for lg, lg_tile in ((6, 8), (6, 11), (9, 10)):
            _check(oracle, emu, field, _matrix(field, lg, width, width + lg), lg, lg_tile,
                   ALL if lg == 6 and lg_tile == 8 else SOME)


@pytest.mark.parametrize("lg,split,lg_tile,width", [
    (6, "2,2,2", 6, 5), (9, "3,3,3", 6, 3), (9, "1,1,7", 8, 9), (10, "4,3,3", 7, 4), (13, "5,4,4", 9, 3),
    (12, "4,8", 10, 7),
    # the shapes with a statically shaped kernel: (12, 2), (11, 3), (10, 4), (10, 3), (8, 4)
    (14, "12,2", 14, 5), (13, "11,2", 14, 9), (14, "10,4", 14, 17), (13, "10,3", 13, 8), (12, "8,4", 12, 16)])
def test_matrix_forced_split(oracle, emu, lg, split, lg_tile, width, monkeypatch):
    """multi-pass plans chosen through SPPARK_B200_NTT_SPLIT (scratch ping-pong for NN / BB)"""
    monkeypatch.setenv("SPPARK_B200_NTT_SPLIT", split)
    combos = ALL if (width << lg) <= 1 << 14 else SOME
    for field in (0, 1):
        _check(oracle, emu, field, _matrix(field, lg, width, 31 * lg + field), lg, lg_tile, combos)


def _loose(n, seed):
    """Goldilocks words that reach the carry corners of add/sub: [p, 2^64), [0, 2^32), corners, canonical"""
    rng = np.random.default_rng(seed)
    high = np.uint64(GL_P) + rng.integers(0, 2**32 - 1, size=n, dtype=np.uint64)
    low = rng.integers(0, 2**32, size=n, dtype=np.uint64)
    canon = rng.integers(0, GL_P, size=n, dtype=np.uint64)
    corners = np.array([0, 1, GL_P - 1, GL_P, GL_P + 1, 2**64 - 1], dtype=np.uint64)
    corner = corners[rng.integers(0, len(corners), size=n)]
    return np.choose(rng.integers(0, 4, size=n), [high, low, canon, corner])


@pytest.mark.parametrize("lg,split,lg_tile,width", [(1, None, 14, 3), (3, None, 14, 5), (8, None, 7, 9),
                                                     (10, "4,3,3", 8, 5), (12, "12", 14, 4)])
def test_matrix_loose_goldilocks_words(oracle, emu, lg, split, lg_tile, width, monkeypatch):
    """any uint64 is a Goldilocks input word and stands for its value mod p; outputs are canonical"""
    if split:
        monkeypatch.setenv("SPPARK_B200_NTT_SPLIT", split)
    else:
        monkeypatch.delenv("SPPARK_B200_NTT_SPLIT", raising=False)
    x = _loose((1 << lg) * width, lg).reshape(1 << lg, width)
    reduced = np.where(x >= np.uint64(GL_P), x - np.uint64(GL_P), x)
    _check(oracle, emu, 0, x, lg, lg_tile, ALL, reduced)


@pytest.mark.parametrize("lg,lb,width,lg_tile", [(1, 1, 3, 14), (4, 2, 1, 14), (5, 3, 9, 7), (7, 1, 4, 8),
                                                 (10, 2, 3, 9)])
@pytest.mark.parametrize("field", [0, 1])
def test_matrix_lde_matches_oracle(oracle, emu, field, lg, lb, width, lg_tile, monkeypatch):
    """inverse NR, the spread with the coset shift, forward RN: every column of d_out is the oracle's
    LDE of that column, and d_in holds its coefficients in bit-reversed row order"""
    monkeypatch.delenv("SPPARK_B200_NTT_SPLIT", raising=False)
    x = _matrix(field, lg, width, 7 * lg + lb)
    d_in = x.copy()
    d_out = np.full(((1 << lg) << lb, width), 12345, dtype=x.dtype)
    assert emu.emu_lde_matrix(field, d_out.ctypes.data, d_in.ctypes.data, lg, lb, width, lg_tile) >= 1
    idx = _brev_idx(lg)
    name = "gl64" if field == 0 else "bb31"
    for c in range(width):
        ext, coef = oracle.lde(name, np.ascontiguousarray(x[:, c]), lb)
        assert np.array_equal(d_out[:, c], ext), (field, lg, lb, c)
        assert np.array_equal(d_in[:, c], coef[idx]), (field, lg, lb, c)


def test_matrix_tile_shapes(emu, monkeypatch):
    """(rows, adjacent matrix columns) of every pass at the full 2^14-element tile: two passes up to
    2^24, the columns filling the tile next to the rows, never more than the width needs, at most 64"""
    monkeypatch.delenv("SPPARK_B200_NTT_SPLIT", raising=False)

    def shapes(lg, width, lg_tile=14, order=NN):
        out, p = [], 0
        while (v := emu.emu_matrix_shape(lg, width, order, lg_tile, p)) >= 0:
            out.append((v >> 8, v & 255))
            p += 1
        return out
    assert shapes(24, 16) == [(12, 2), (12, 2)]
    assert shapes(22, 64) == [(11, 3), (11, 3)]
    assert shapes(20, 256) == [(10, 4), (10, 4)]
    assert shapes(20, 8) == [(10, 3), (10, 3)]
    assert shapes(20, 1) == [(10, 0), (10, 0)]
    assert shapes(3, 1000) == [(3, 6)]
    assert shapes(27, 5, order=RN) == [(9, 3), (9, 3), (9, 3)]


def test_set_matrix_refuses_other_plans(emu):
    """plans with several transform columns per tile, or slab routing, have no matrix form"""
    assert emu.emu_matrix_rejects() == 1


def _no_gpu():
    import torch
    return not torch.cuda.is_available()


def test_matrix_entry_points_without_device(lib):
    """no CPU fallback: every matrix entry point returns -cudaErrorNoDevice (-100) and leaves the
    caller's memory as it was"""
    if not _no_gpu():
        pytest.skip("a GPU is present; the failure path is exercised on CPU-only hosts")
    for field, dt in ((0, np.uint64), (1, np.uint32)):
        buf = np.arange(8 * 5, dtype=dt)
        before = buf.copy()
        out = np.zeros(16 * 5, dtype=dt)
        errs = [lib.sppark_b200_ntt_matrix(field, 0, buf.ctypes.data, 3, 5, 0, 0, 0),
                lib.sppark_b200_ntt_matrix_dev(field, buf.ctypes.data, 3, 5, 0, 0, 0, None),
                lib.sppark_b200_lde_matrix_dev(field, out.ctypes.data, buf.ctypes.data, 3, 1, 5, None)]
        for e in errs:
            assert e.code == -100
            if e.message:
                lib.drop_error_message(e.message)
        assert np.array_equal(buf, before) and not out.any()


def test_matrix_entry_points_refuse_before_any_work(lib):
    """256-bit fields, unknown fields, bad orders and out-of-range sizes are -cudaErrorInvalidValue
    on any host, before a device is looked for"""
    buf = np.arange(8 * 5, dtype=np.uint64)
    before = buf.copy()
    out = np.zeros(16 * 5, dtype=np.uint64)
    errs = [lib.sppark_b200_ntt_matrix(2, 0, buf.ctypes.data, 3, 5, 0, 0, 0),            # BLS12-381 Fr
            lib.sppark_b200_ntt_matrix_dev(5, buf.ctypes.data, 3, 5, 0, 0, 0, None),     # BN254 Fr
            lib.sppark_b200_lde_matrix_dev(6, out.ctypes.data, buf.ctypes.data, 3, 1, 5, None),
            lib.sppark_b200_ntt_matrix(9, 0, buf.ctypes.data, 3, 5, 0, 0, 0),            # unknown field
            lib.sppark_b200_ntt_matrix(0, 0, buf.ctypes.data, 3, 5, 5, 0, 0),            # order 5
            lib.sppark_b200_ntt_matrix_dev(0, buf.ctypes.data, 3, 5, 0, 2, 0, None),     # direction 2
            lib.sppark_b200_ntt_matrix(1, 0, buf.ctypes.data, 28, 5, 0, 0, 0),           # 2^28 BabyBear
            lib.sppark_b200_ntt_matrix(0, 0, buf.ctypes.data, 30, 1 << 40, 0, 0, 0)]     # size_t overflow
    msgs = []
    for e in errs:
        assert e.code == -1
        msgs.append(C.cast(e.message, C.c_char_p).value.decode() if e.message else "")
        if e.message:
            lib.drop_error_message(e.message)
    assert "Goldilocks and BabyBear only" in msgs[0] and "Goldilocks and BabyBear only" in msgs[2]
    assert "unknown field" in msgs[3]
    assert np.array_equal(buf, before) and not out.any()
    # lg 0 and width 0 are no-ops that succeed
    assert lib.sppark_b200_ntt_matrix(0, 0, buf.ctypes.data, 0, 5, 0, 0, 0).code == 0
    assert lib.sppark_b200_ntt_matrix(0, 0, buf.ctypes.data, 3, 0, 0, 0, 0).code == 0
    assert np.array_equal(buf, before)


def test_matrix_wrappers_validate_shapes(lib):
    """shape, rank, element-size / field mismatches and 256-bit field ids are ValueError, raised
    before the library is called"""
    from sppark_b200 import ntt
    with pytest.raises(ValueError):
        ntt.ntt_matrix(0, np.zeros((6, 3), dtype=np.uint64))               # height not a power of two
    with pytest.raises(ValueError):
        ntt.ntt_matrix(0, np.zeros(8, dtype=np.uint64))                    # rank 1
    with pytest.raises(ValueError):
        ntt.ntt_matrix(0, np.zeros((8, 3, 4), dtype=np.uint64))            # rank 3
    with pytest.raises(ValueError):
        ntt.ntt_matrix(0, np.zeros((8, 3), dtype=np.uint32), field=ntt.GL64)
    with pytest.raises(ValueError):
        ntt.ntt_matrix(0, np.zeros((8, 3), dtype=np.uint64), field=ntt.BB31)
    with pytest.raises(ValueError):
        ntt.ntt_matrix(0, np.zeros((8, 3), dtype=np.uint64), field=ntt.BLS12_381_FR)
    with pytest.raises(ValueError):
        ntt.ntt_matrix(0, np.zeros((8, 3), dtype=np.float32))
    with pytest.raises(ValueError):
        ntt.ntt_matrix(0, np.zeros((3, 8), dtype=np.uint64).T)             # not C-contiguous
    if _no_gpu():
        from sppark_b200 import _lib
        with pytest.raises(_lib.SpparkError):
            ntt.ntt_matrix(0, np.zeros((8, 3), dtype=np.uint64))          # well-formed: reaches the library
