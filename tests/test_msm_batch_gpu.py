"""Batched MSM on the device (MsmContext.invoke_batch / sppark_b200_msm_ctx_invoke_batch, msm_dev_batch /
sppark_b200_msm_dev_batch): every vector's result against a loop of the single entries on the same
inputs (ctx_invoke_bits / msm_dev_bits), and against the oracle at small sizes, as affine points; the
group geometry from the SPPARK_B200_MSM_DEBUG lines (sets = G V); the refusals.

Inputs as in test_msm_geometry_gpu.py: m distinct points repeated (one at infinity, one the negation of
its neighbour)."""
import re

import numpy as np
import pytest

from test_msm_geometry_gpu import _curve

pytestmark = pytest.mark.gpu

CURVES = ["bls12_381", "pallas", "vesta", "bn254", "bls12_377", "bls12_381_g2", "bn254_g2", "bls12_377_g2"]
LINE = re.compile(r"\[msm\] slice \d+ n=(\d+) wbits=(\d+) nwins=\d+ .*? digits=(\d+) sets=(\d+) copies=(\d+) "
                  r"nbits=\d+ sbytes=\d+ vecs=(\d+) vsets=(\d+)")
INVALID = -1


@pytest.fixture
def debug(monkeypatch, capfd):
    monkeypatch.setenv("SPPARK_B200_MSM_DEBUG", "1")
    for k in ("SPPARK_B200_MSM_WBITS", "SPPARK_B200_MSM_HEAVY", "SPPARK_B200_MSM_SLICES", "SPPARK_B200_MSM_SCHED",
              "SPPARK_B200_MSM_PAIR", "SPPARK_B200_MSM_BATCH_GROUP"):
        monkeypatch.delenv(k, raising=False)
    capfd.readouterr()
    return capfd


def _groups(capfd):
    """(n, wbits, digits, sets, copies, vecs, vsets) per debug line since the last read"""
    return [tuple(map(int, t)) for t in LINE.findall(capfd.readouterr().err)]


def _points(c, n, m=64):
    base = c.base(min(m, max(n, 1)))
    return np.ascontiguousarray(base[np.arange(n) % base.shape[0]])


def _scalars(B, n, seed, r):
    """(B, n, 4) uint64 below r, with a few r - 1 and zeros"""
    rng = np.random.default_rng(seed)
    sc = rng.integers(0, 2**63, size=(B, n, 4), dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, size=(B, n, 4),
                                                                                             dtype=np.uint64)
    top = np.uint64(r >> 192)
    sc[:, :, 3] %= top
    if n > 2:
        rm1 = [(r - 1) >> (64 * i) & (2**64 - 1) for i in range(4)]
        sc[:, 1] = rm1
        sc[:, 2] = 0
    return sc


def _same(c, a, b):
    return np.array_equal(c.affine(a), c.affine(b))


def _ctx(c, pts, K=None):
    from sppark_b200 import msm
    return msm.MsmContext(c.cid, pts, precompute=K)


def _check_ctx(c, ctx, sc, nbits=None):
    """invoke_batch against a loop of invoke (32-byte scalars) / invoke_bits, row by row"""
    got = ctx.invoke_batch(sc, nbits=nbits)
    assert got.shape == (sc.shape[0], 3 * (got.shape[1] // 3))
    for b in range(sc.shape[0]):
        assert _same(c, got[b], ctx.invoke(np.ascontiguousarray(sc[b]), nbits=nbits)), (c.name, b, sc.shape)
    return got


@pytest.mark.parametrize("curve", CURVES)
@pytest.mark.parametrize("n", [1, 31, 1 << 10, 1 << 16])
def test_batch_matches_single_calls(oracle, curve, n):
    c = _curve(oracle, curve)
    pts = _points(c, n)
    ctx = _ctx(c, pts)
    for B in (1, 2, 7, 33):
        _check_ctx(c, ctx, _scalars(B, n, n + B, c.r))
    ctx.close()


@pytest.mark.parametrize("curve", CURVES)
def test_batch_matches_oracle(oracle, curve):
    c = _curve(oracle, curve)
    n = 31
    pts = _points(c, n, m=n)
    sc = _scalars(3, n, 5, c.r)
    ctx = _ctx(c, pts)
    got = ctx.invoke_batch(sc)
    for b in range(3):
        assert np.array_equal(c.affine(got[b]), c.reference(pts, sc[b])), (curve, b)
    ctx.close()


@pytest.mark.parametrize("curve", CURVES)
@pytest.mark.parametrize("K", [4, 64])
def test_batch_precomputed(oracle, debug, curve, K):
    """tables of K = 4 copies and of K = D (every digit its own copy); the batch invokes fewer points than
    the context holds"""
    c = _curve(oracle, curve)
    N = 1 << 10
    pts = _points(c, N)
    ctx = _ctx(c, pts, K)
    debug.readouterr()
    for n, B in ((N, 5), (1000, 7), (31, 2)):
        sc = _scalars(B, n, K + n, c.r)
        _check_ctx(c, ctx, sc)
        lines = _groups(debug)
        batch_line = lines[0]
        n_, wbits, digits, sets, copies, vecs, vsets = batch_line
        assert (n_, vecs, sets) == (n, B, B * vsets) and copies == -(-digits // vsets), batch_line
        assert all(l[5] == 1 and l[3] == vsets for l in lines[1:]), lines
    ctx.close()


@pytest.mark.parametrize("sbytes,nbits", [(4, 32), (4, 16), (8, 64), (16, 128), (32, 200)])
def test_batch_small_scalars_pinned_and_pageable(oracle, sbytes, nbits):
    """host scalars of every width, from pageable and from pinned memory"""
    import torch
    c = _curve(oracle, "bls12_381")
    n, B = 3000, 6
    pts = _points(c, n)
    ctx = _ctx(c, pts)
    rng = np.random.default_rng(sbytes + nbits)
    words = rng.integers(0, 2**32, size=(B, n * sbytes // 4), dtype=np.uint64).astype(np.uint32)
    if sbytes == 4:
        sc = words.reshape(B, n)
    elif sbytes == 8:
        sc = words.view(np.uint64).reshape(B, n)
    else:
        sc = words.view(np.uint64).reshape(B, n, sbytes // 8)
    sc = np.ascontiguousarray(sc)
    want = _check_ctx(c, ctx, sc, nbits)
    pinned = torch.from_numpy(sc.view(np.uint8).reshape(-1).copy()).pin_memory()
    psc = pinned.numpy().view(sc.dtype).reshape(sc.shape)
    got = ctx.invoke_batch(psc, nbits=nbits)
    assert all(_same(c, got[b], want[b]) for b in range(B))
    ctx.close()


@pytest.mark.parametrize("curve", ["bls12_381", "bn254_g2"])
def test_dev_batch_side_stream(oracle, curve):
    import torch
    from sppark_b200 import msm
    c = _curve(oracle, curve)
    n, B = 5000, 7
    pts = _points(c, n)
    sc = _scalars(B, n, 9, c.r)
    d_pts = torch.from_numpy(pts.view(np.int64)).cuda()
    d_sc = torch.from_numpy(sc.view(np.int64)).cuda()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        got = msm.msm_dev_batch(c.cid, d_pts, d_sc, stream=side.cuda_stream)
    for b in range(B):
        assert _same(c, got[b], msm.msm_dev(c.cid, d_pts, d_sc[b].contiguous())), b
    # 8-byte scalars with a bound, against msm_dev_bits
    d8 = torch.from_numpy(sc[:, :, 0].copy().view(np.int64)).cuda()
    got = msm.msm_dev_batch(c.cid, d_pts, d8, nbits=40)
    for b in range(B):
        assert _same(c, got[b], msm.msm_dev(c.cid, d_pts, d8[b].contiguous(), nbits=40)), b


def test_forced_group_sizes(oracle, debug, monkeypatch):
    """7 vectors in groups of 3 (3 + 3 + 1: a short last group), of 1 and of all 7, on host and device"""
    import torch
    from sppark_b200 import msm
    c = _curve(oracle, "bls12_381")
    n, B = 2000, 7
    pts = _points(c, n)
    sc = _scalars(B, n, 3, c.r)
    ctx = _ctx(c, pts)
    want = ctx.invoke_batch(sc)
    d_pts, d_sc = torch.from_numpy(pts.view(np.int64)).cuda(), torch.from_numpy(sc.view(np.int64)).cuda()
    for G, vecs in ((3, [3, 3, 1]), (1, [1] * 7), (7, [7]), (100, [7])):
        monkeypatch.setenv("SPPARK_B200_MSM_BATCH_GROUP", str(G))
        debug.readouterr()
        for run in (lambda: ctx.invoke_batch(sc), lambda: msm.msm_dev_batch(c.cid, d_pts, d_sc)):
            got = run()
            assert all(_same(c, got[b], want[b]) for b in range(B)), G
            lines = _groups(debug)
            assert [l[5] for l in lines] == vecs and all(l[3] == l[5] * l[6] for l in lines), (G, lines)
    ctx.close()


def test_default_group_holds_a_small_batch(oracle, debug):
    """without the override, 33 vectors of 2^12 points run as one group of 33 V sets"""
    c = _curve(oracle, "bls12_381")
    n, B = 1 << 12, 33
    ctx = _ctx(c, _points(c, n))
    ctx.invoke_batch(_scalars(B, n, 1, c.r))
    lines = _groups(debug)
    assert len(lines) == 1 and lines[0][5] == B and lines[0][3] == B * lines[0][6], lines
    ctx.close()


def test_bls12_381_2pow20_by_16(oracle):
    c = _curve(oracle, "bls12_381")
    n, B = 1 << 20, 16
    pts = _points(c, n, m=2048)
    ctx = _ctx(c, pts)
    _check_ctx(c, ctx, _scalars(B, n, 20, c.r))
    ctx.close()


def test_edge_cases_and_refusals(oracle):
    import torch
    from sppark_b200 import _lib, msm
    c = _curve(oracle, "bls12_381")
    pts = _points(c, 100)
    ctx = _ctx(c, pts)
    assert not ctx.invoke_batch(np.zeros((4, 0, 4), dtype=np.uint64)).any()        # npoints == 0: infinities
    assert ctx.invoke_batch(np.zeros((0, 100, 4), dtype=np.uint64)).shape == (0, 18)
    with pytest.raises(_lib.SpparkError):
        ctx.invoke_batch(np.zeros((2, 101, 4), dtype=np.uint64))                   # more than preloaded
    l = _lib.lib()
    out = np.ones((2, 18), dtype=np.uint64)
    sc = np.zeros(2 * 101 * 8, dtype=np.uint64)
    err = l.sppark_b200_msm_ctx_invoke_batch(ctx._h, out.ctypes.data, sc.ctypes.data, 101, 2, 32, 255)
    assert err.code == INVALID and not out.any()
    l.drop_error_message(err.message)
    out = np.ones((2, 18), dtype=np.uint64)
    err = l.sppark_b200_msm_ctx_invoke_batch(ctx._h, out.ctypes.data, sc.ctypes.data, 10, 2, 12, 8)
    assert err.code == INVALID and not out.any()
    l.drop_error_message(err.message)
    d_pts = torch.from_numpy(pts.view(np.int64)).cuda()
    d_sc = torch.zeros(2 * 100 * 4 + 2, dtype=torch.int64, device="cuda")
    for off in (4, 8):                                                               # misaligned for 16/32 bytes
        out = np.ones((2, 18), dtype=np.uint64)
        err = l.sppark_b200_msm_dev_batch(0, out.ctypes.data, d_pts.data_ptr(), 100, d_sc.data_ptr() + off, 2, 32, 255,
                                          None)
        assert err.code == INVALID and not out.any(), off
        l.drop_error_message(err.message)
    out = np.ones((2, 18), dtype=np.uint64)
    assert l.sppark_b200_msm_dev_batch(0, out.ctypes.data, d_pts.data_ptr(), 0, d_sc.data_ptr(), 2, 32, 255,
                                       None).code == 0
    assert not out.any()
    ctx.close()
