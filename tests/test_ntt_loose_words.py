"""Goldilocks NTT on non-canonical input words, on the CPU single-stepper (tests/emu/ntt_emu.cpp,
the HD pass code of ntt_core.cuh run phase by phase): any uint64 is a legal input word and stands
for its value mod p, and every output word is canonical.  Each transform is compared bit-exactly
with the oracle on the reduced input x % p."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

P = 2**64 - 2**32 + 1
EMU_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu", "ntt_emu.cpp")
CORNERS = np.array([0, 1, P - 1, P, P + 1, 2**64 - 1], dtype=np.uint64)


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("ntt_emu") / "libntt_emu.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-x", "c++", "-o", so, EMU_SRC])
    l = C.CDLL(so)
    l.emu_ntt_gl64.argtypes = [C.c_void_p, C.c_uint, C.c_int, C.c_int, C.c_uint]
    l.emu_ntt_slab_gl64.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_uint, C.c_uint, C.c_uint, C.c_int, C.c_uint]
    l.emu_ntt_slab_p2p_gl64.argtypes = [C.c_void_p, C.c_void_p, C.c_uint, C.c_uint, C.c_uint, C.c_int, C.c_uint]
    return l


def loose_words(n, seed, pattern="mixed"):
    """Words that reach the carry corners of add/sub: a mix of [p, 2^64), [0, 2^32), the corners
    and canonical words; 'high' makes every word >= p (first-stage partners both large), 'top' /
    'bottom' the first / second half only, with small words in the other half."""
    rng = np.random.default_rng(seed)
    high = np.uint64(P) + rng.integers(0, 2**32 - 1, size=n, dtype=np.uint64)      # [p, 2^64)
    low = rng.integers(0, 2**32, size=n, dtype=np.uint64)
    if pattern == "high":
        return high
    if pattern in ("top", "bottom"):
        h = n // 2
        return np.concatenate([high[:h], low[h:]] if pattern == "top" else [low[:h], high[h:]])
    canon = rng.integers(0, P, size=n, dtype=np.uint64)
    corner = CORNERS[rng.integers(0, len(CORNERS), size=n)]
    return np.choose(rng.integers(0, 4, size=n), [high, low, canon, corner])


PATTERNS = ["mixed", "high", "top", "bottom"]


def _reduce(x):
    return np.where(x >= np.uint64(P), x - np.uint64(P), x)


def test_known_answer_lg1(emu):
    """[2^64 - 1, 2^64 - 1] is [2^32 - 2, 2^32 - 2] mod p: its 2-point DFT is [2^33 - 4, 0]"""
    y = np.array([2**64 - 1, 2**64 - 1], dtype=np.uint64)
    emu.emu_ntt_gl64(y.ctypes.data, 1, 0, 0, 14)
    assert y.tolist() == [0x1FFFFFFFC, 0]


def test_generator_reaches_the_bad_carries():
    """the inputs above must actually hold pairs whose unreduced sum wraps twice and pairs whose
    difference borrows twice, or the tests below could not fail"""
    x = [int(v) for v in loose_words(1 << 10, 0, "mixed")]
    h = [int(v) for v in loose_words(1 << 10, 0, "high")]
    assert any(a + b >= 2**65 - 2**32 + 1 for a, b in zip(h[:512], h[512:]))     # add: 2^64 + EPS wraps
    assert any(b > a + P for a, b in zip(x, x[1:]))                              # sub: a - b + 2^64 < EPS


# the sizes and digit splits of test_emu.py's planner cases, up to 2^13
CASES = [(lg, None) for lg in range(1, 14)] + [
    (6, "2,2,2"), (6, "1,5"), (6, "5,1"), (9, "3,3,3"), (9, "4,2,3"), (9, "1,1,7"), (9, "7,1,1"),
    (9, "2,2,2,3"), (13, "5,4,4"), (13, "6,7"), (10, "4,3,3"), (10, "3,7")]


@pytest.mark.parametrize("lg,split", CASES)
def test_block_pass_loose_inputs(oracle, emu, lg, split, monkeypatch):
    if split:
        monkeypatch.setenv("SPPARK_B200_NTT_SPLIT", split)
    else:
        monkeypatch.delenv("SPPARK_B200_NTT_SPLIT", raising=False)
    for k, pattern in enumerate(PATTERNS):
        x = loose_words(1 << lg, 16 * lg + k, pattern)
        xr = _reduce(x)
        for order in range(5):                          # NN, NR, RN, RR and BB (bit-reversed in and out)
            for inv in (0, 1):
                want = oracle.ntt_gl64(xr, order, bool(inv))
                for lg_tile in (14, 7):
                    y = x.copy()
                    emu.emu_ntt_gl64(y.ctypes.data, lg, order, inv, lg_tile)
                    assert (y < np.uint64(P)).all(), (pattern, order, inv, lg_tile)
                    assert np.array_equal(y, want), (pattern, order, inv, lg_tile)


@pytest.mark.parametrize("lg,lg_g,split,lg_tile", [(4, 1, None, 14), (8, 3, None, 6), (10, 3, None, 14),
                                                   (12, 0, None, 14), (9, 3, "3,3,3", 14), (11, 2, "3,4,4", 7)])
def test_slab_passes_loose_inputs(oracle, emu, lg, lg_g, split, lg_tile, monkeypatch):
    """the slab-sharded transform's first stage reads the caller's words: staging route and
    fused-exchange route, G ranks simulated in one process"""
    from sppark_b200 import parallel
    if split:
        monkeypatch.setenv("SPPARK_B200_NTT_SPLIT", split)
    else:
        monkeypatch.delenv("SPPARK_B200_NTT_SPLIT", raising=False)
    s1 = int(split.split(",")[0]) if split else None
    G = 1 << lg_g
    for k, pattern in enumerate(PATTERNS):
        x = loose_words(1 << lg, 64 * lg + 8 * lg_g + k, pattern)
        for inv in (0, 1):
            want = oracle.ntt_gl64(_reduce(x), 0, bool(inv))
            stag = []
            for r in range(G):
                loc = parallel.scatter_columns(x, lg, lg_g, r, s1=s1).reshape(-1).copy()
                st = np.zeros_like(loc)
                assert emu.emu_ntt_slab_gl64(1, loc.ctypes.data, st.ctypes.data, lg, lg_g, r, inv, lg_tile) == 0
                stag.append(st.reshape(G, -1))
            staged = [np.concatenate([stag[q][r] for q in range(G)]).copy() for r in range(G)]
            fused = [np.zeros((1 << lg) // G, dtype=np.uint64) for _ in range(G)]
            ptrs = (C.c_void_p * G)(*[f.ctypes.data for f in fused])
            for r in range(G):
                loc = parallel.scatter_columns(x, lg, lg_g, r, s1=s1).reshape(-1).copy()
                assert emu.emu_ntt_slab_p2p_gl64(loc.ctypes.data, ptrs, lg, lg_g, r, inv, lg_tile) == 0
            for route, recv in (("staging", staged), ("fused", fused)):
                for r in range(G):
                    scratch = np.zeros_like(recv[r])
                    assert emu.emu_ntt_slab_gl64(2, recv[r].ctypes.data, scratch.ctypes.data, lg, lg_g, r, inv, lg_tile) == 0
                got = parallel.gather_columns(recv, lg, lg_g, s1=s1)
                assert (got < np.uint64(P)).all(), (route, pattern, inv)
                assert np.array_equal(got, want), (route, pattern, inv)
