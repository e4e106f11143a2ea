"""Batched NTT without a GPU: the batched pass descriptors (make_plan + set_batch) run through the
HD phase functions of ntt_core.cuh by the CPU single-stepper tests/emu/ntt_batch_emu.cpp; every
row must equal the oracle's transform of that row.  Also: the batched C entry points and Python
wrappers fail cleanly on a CPU-only host."""
import ctypes as C
import os
import random
import subprocess

import numpy as np
import pytest

EMU = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu")
GL_P = 2**64 - 2**32 + 1
BB_P = 0x78000001
NN, NR, RN, RR, BB = range(5)


@pytest.fixture(scope="module")
def emu():
    so, src = os.path.join(EMU, "libntt_batch_emu.so"), os.path.join(EMU, "ntt_batch_emu.cpp")
    csrc = os.path.join(os.path.dirname(EMU), "..", "sppark_b200", "csrc")
    newest = max(os.path.getmtime(os.path.join(r, f)) for r, _, fs in os.walk(csrc) for f in fs)
    if not os.path.exists(so) or os.path.getmtime(so) < max(newest, os.path.getmtime(src)):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-x", "c++", "-o", so, src])
    l = C.CDLL(so)
    l.emu_ntt_batch.argtypes = [C.c_int, C.c_void_p, C.c_uint, C.c_size_t, C.c_int, C.c_int, C.c_int, C.c_uint]
    return l


def _brev_rows(a, lg):
    idx = np.array([int(format(i, f"0{lg}b")[::-1], 2) for i in range(1 << lg)]) if lg else np.zeros(1, int)
    return a[idx]


def _oracle_row(ofn, x, lg, order, inv, coset):
    """oracle transform of one row; the oracle has no coset BB, which is bitrev(coset NN(bitrev x))"""
    if coset and order == BB:
        return _brev_rows(ofn(_brev_rows(x, lg), NN, bool(inv), True), lg)
    return ofn(x, order, bool(inv), bool(coset))


def _check(oracle, emu, field, lg, batch, lg_tile, seed, types=(0, 1)):
    rng = np.random.default_rng(seed)
    if field == 0:
        x = rng.integers(0, GL_P, size=(batch, 1 << lg), dtype=np.uint64)
        ofn = oracle.ntt_gl64
    elif field == 1:
        x = rng.integers(0, BB_P, size=(batch, 1 << lg), dtype=np.uint32)
        ofn = oracle.ntt_bb31
    else:
        rnd = random.Random(seed)
        p = oracle.ff_consts("bls12_381_fr")["p"]
        x = np.array([[oracle.int_to_limbs(rnd.randrange(p), 4) for _ in range(1 << lg)] for _ in range(batch)],
                     dtype=np.uint64)
        ofn = lambda a, *k: oracle.ntt_ff("bls12_381_fr", a, *k)   # noqa: E731
    for order in range(5):
        for inv in (0, 1):
            for coset in types:
                y = x.copy()
                assert emu.emu_ntt_batch(field, y.ctypes.data, lg, batch, order, inv, coset, lg_tile) >= 1
                for b in range(batch):
                    want = _oracle_row(ofn, x[b], lg, order, inv, coset)
                    assert np.array_equal(y[b], want), (field, lg, batch, order, inv, coset, b)


@pytest.mark.parametrize("lg", range(1, 15))
@pytest.mark.parametrize("field", [0, 1])
def test_batch_rows_match_oracle(oracle, emu, field, lg, monkeypatch):
    """every lg of 1..14 with a batch of {1, 2, 3, 5, 8}, and 2^7-element tiles so that the
    transforms of 2^8 and more span several tiles"""
    monkeypatch.delenv("SPPARK_B200_NTT_SPLIT", raising=False)
    batch = (1, 2, 3, 5, 8)[lg % 5]
    _check(oracle, emu, field, lg, batch, 7 if lg > 4 else 14, 1000 * field + lg)


@pytest.mark.parametrize("batch", [1, 2, 3, 5, 8])
def test_batch_sizes_small_transforms(oracle, emu, batch, monkeypatch):
    """one-tile transforms (a tile per row) and two-tile ones at every batch size"""
    monkeypatch.delenv("SPPARK_B200_NTT_SPLIT", raising=False)
    for field in (0, 1):
        for lg, lg_tile in ((3, 14), (6, 5)):
            _check(oracle, emu, field, lg, batch, lg_tile, 17 * batch + lg)


@pytest.mark.parametrize("lg,split", [(6, "2,2,2"), (9, "3,3,3"), (9, "1,1,7"), (10, "4,3,3"), (13, "5,4,4"),
                                      (12, "4,8")])
def test_batch_forced_multipass(oracle, emu, lg, split, monkeypatch):
    """multi-pass plans (scratch ping-pong of batch x 2^lg elements for NN / BB) with small tiles"""
    monkeypatch.setenv("SPPARK_B200_NTT_SPLIT", split)
    for field in (0, 1):
        _check(oracle, emu, field, lg, 3 if lg < 12 else 2, 6, 31 * lg + field)


@pytest.mark.parametrize("lg,batch,lg_tile", [(1, 3, 11), (4, 5, 11), (8, 2, 5), (11, 3, 11), (12, 2, 8)])
def test_batch_256bit(oracle, emu, lg, batch, lg_tile, monkeypatch):
    monkeypatch.delenv("SPPARK_B200_NTT_SPLIT", raising=False)
    _check(oracle, emu, 2, lg, batch, lg_tile, lg, types=(0, 1) if lg <= 8 else (0,))


def test_set_batch_rejects_slab_passes(emu):
    assert emu.emu_batch_rejects_slab() == 1


def _no_gpu():
    import torch
    return not torch.cuda.is_available()


def test_batch_entry_points_without_device(lib):
    """no CPU fallback: every batched entry point returns -cudaErrorNoDevice (-100) and leaves the
    caller's memory as it was"""
    if not _no_gpu():
        pytest.skip("a GPU is present; the failure path is exercised on CPU-only hosts")
    for field, dt in ((0, np.uint64), (1, np.uint32)):
        buf = np.arange(4 * 8, dtype=dt)
        before = buf.copy()
        out = np.zeros(4 * 16, dtype=dt)
        errs = [lib.sppark_b200_ntt_batch(field, 0, buf.ctypes.data, 3, 4, 0, 0, 0),
                lib.sppark_b200_ntt_batch_dev(field, buf.ctypes.data, 3, 4, 0, 0, 0, None),
                lib.sppark_b200_lde_batch_dev(field, out.ctypes.data, buf.ctypes.data, 3, 1, 4, None)]
        for e in errs:
            assert e.code == -100
            if e.message:
                lib.drop_error_message(e.message)
        assert np.array_equal(buf, before) and not out.any()


def test_batch_wrappers_validate_shapes(lib):
    """shape errors are ValueError, raised before the library is called"""
    from sppark_b200 import ntt
    with pytest.raises(ValueError):
        ntt.ntt_batch(0, np.zeros((3, 6), dtype=np.uint64))          # row length not a power of two
    with pytest.raises(ValueError):
        ntt.ntt_batch(0, np.zeros(8, dtype=np.uint64))               # rank 1
    with pytest.raises(ValueError):
        ntt.ntt_batch(0, np.zeros((2, 8), dtype=np.uint64), field=ntt.BLS12_381_FR)   # needs (batch, n, 4)
    with pytest.raises(ValueError):
        ntt.ntt_batch(0, np.zeros((2, 8, 3), dtype=np.uint64), field=ntt.BLS12_381_FR)
    with pytest.raises(ValueError):
        ntt.ntt_batch(0, np.zeros((2, 8), dtype=np.uint32), field=ntt.GL64)    # 4-byte words, 8-byte field
    with pytest.raises(ValueError):
        ntt.ntt_batch(0, np.zeros((2, 8), dtype=np.uint64), field=ntt.BB31)
    with pytest.raises(ValueError):
        ntt.ntt_batch(0, np.zeros((2, 8, 4), dtype=np.uint32), field=ntt.BLS12_381_FR)
    if _no_gpu():
        from sppark_b200 import _lib
        with pytest.raises(_lib.SpparkError):
            ntt.ntt_batch(0, np.zeros((2, 8), dtype=np.uint64))       # well-formed: reaches the library
