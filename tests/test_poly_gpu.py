"""Parity of the polynomial helpers (SURVEY.md section 8 row f4) with the oracle and with the
recordings of the reference's own kernels -- through the C ABI (sppark_b200/poly.py is a thin
ctypes wrapper over sppark_b200_{prefix_op,div_by_x_minus_z,evaluate,batch_inverse}_dev)."""
import os
import random

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
WORD_FIELDS = ["gl64", "bb31"]
WIDE_FIELDS = ["bls12_381_fr", "pallas_fr", "vesta_fr", "bn254_fr", "bls12_377_fr"]


def _vals(field, n, seed):
    from oracle import poly as op
    rnd = random.Random(seed)
    p = op.FIELDS[field]["p"]
    return [rnd.randrange(p) for _ in range(n)]


def _fid(field):
    from oracle import poly as op
    return op.FIELDS[field]["id"]


def _sha(a):
    import hashlib
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), dtype=np.uint8)


@pytest.mark.parametrize("field", ["gl64", "bb31", "bls12_381_fr"])
def test_matches_the_reference_recordings(field):
    """every input/output pair tests/golden/make_golden.py recorded from the reference's own
    kernels (what the reference cannot run -- see gen_poly -- is absent from the file);
    the `big` case is compared through SHA-256 digests of whole output arrays"""
    from oracle import poly as op
    from sppark_b200 import poly
    g = np.load(os.path.join(GOLDEN, f"poly_{field}_ref_gpu.npz"))
    fid, big = _fid(field), int(g["big"])
    for n in [int(v) for v in g["lens"]] + [big]:
        x = op.seeded_input(field, n, 4242) if n == big else g[f"in_{n}"]
        same = (lambda a, b: np.array_equal(_sha(a), b)) if n == big else np.array_equal
        y = x.copy()
        poly.prefix_op(poly.ADD, y, field=fid)
        assert same(y, g[f"add_{n}"]), (field, n, "add")
        y = (g[f"mulin_{n}"] if f"mulin_{n}" in g else x).copy()
        poly.prefix_op(poly.MULTIPLY, y, field=fid)
        assert same(y, g[f"mul_{n}"]), (field, n, "mul")
        zs = g[f"z_{n}"]
        ndiv = 0
        for k in range(len(zs)):
            for rot in (0, 1):
                if f"div_{n}_{k}_{rot}" not in g:
                    continue
                y = x.copy()
                poly.div_by_x_minus_z(y, zs[k:k + 1], rotate=bool(rot), field=fid)
                assert same(y, g[f"div_{n}_{k}_{rot}"]), (field, n, k, rot)
                ndiv += 1
        assert ndiv or field == "bls12_381_fr"
        if f"eval_{n}" in g:
            got = poly.evaluate(x, g[f"x_{n}"], field=fid)
            assert np.array_equal(got, g[f"eval_{n}"]), (field, n, "evaluate")


@pytest.mark.parametrize("field,coop", [(f, True) for f in WORD_FIELDS + WIDE_FIELDS] +
                         [("gl64", False), ("bb31", False), ("bls12_381_fr", False)])
def test_matches_oracle(field, coop, monkeypatch):
    """seeded inputs at sizes around every level of the scan hierarchy (thread, warp, tile, many
    tiles) against oracle/poly.py; mid sizes run as one cooperative launch by default and as the
    three-launch scan with SPPARK_B200_POLY_NO_COOP set (what large inputs take) -- both are checked"""
    from oracle import poly as op
    from sppark_b200 import poly
    if not coop:
        monkeypatch.setenv("SPPARK_B200_POLY_NO_COOP", "1")
    p, fid = op.FIELDS[field]["p"], _fid(field)
    wide = field in WIDE_FIELDS
    tile = 1024 if wide else 2048
    lens = [1, 2, 7, 8, 9, 255, 256, 257, tile - 1, tile, tile + 1, 3 * tile + 5]
    lens += [33 * tile + 17] if wide else [33 * tile + 17, 70 * tile + 1]
    for n in lens:
        c = _vals(field, n, 1000 + n)
        if n > 3:
            c[2] = 0
        x = op.encode(field, c)
        y = x.copy()
        poly.prefix_op(poly.ADD, y, field=fid)
        assert np.array_equal(y, op.encode(field, op.prefix_op(p, "add", c))), (field, n, "add")
        cm = [v or 5 for v in c]
        y = op.encode(field, cm)
        poly.prefix_op(poly.MULTIPLY, y, field=fid)
        assert np.array_equal(y, op.encode(field, op.prefix_op(p, "mul", cm))), (field, n, "mul")
        for z in (_vals(field, 1, n)[0], 0, 1, p - 1) if n in (9, tile + 1) else (_vals(field, 1, n)[0],):
            for rot in (False, True):
                y = x.copy()
                poly.div_by_x_minus_z(y, op.encode(field, [z]), rotate=rot, field=fid)
                assert np.array_equal(y, op.encode(field, op.div_by_x_minus_z(p, c, z, rot))), (field, n, z, rot)
        xs = _vals(field, 3, 77 + n) + [0, 1]
        got = poly.evaluate(x, op.encode(field, xs), field=fid)
        assert np.array_equal(got, op.encode(field, op.evaluate(p, c, xs))), (field, n, "evaluate")
        y = x.copy()
        poly.batch_inverse(y, field=fid)
        assert np.array_equal(y, op.encode(field, op.batch_inversion(p, c))), (field, n, "inverse")


def test_prefix_multiply_through_zero():
    """a zero input zeroes every later product (polynomial/prefix_op.cuh Multiply has no special case)"""
    from oracle import poly as op
    from sppark_b200 import poly
    c = _vals("gl64", 5000, 3)
    c[2500] = 0
    y = op.encode("gl64", c)
    poly.prefix_op(poly.MULTIPLY, y)
    assert np.array_equal(y, op.encode("gl64", op.prefix_op(op.GL64_P, "mul", c)))
    assert not y[2500:].any()


@pytest.mark.parametrize("field", WORD_FIELDS)
def test_large_sizes_by_properties(field):
    """2^22 + 3 elements (2049 tiles), checked through size-independent identities:
    p(x) = q(x) (x - z) + r at a random x, r = p(z), prefix-add's last element = the plain sum,
    prefix-multiply of the batch inverses = inverse of the prefix-multiply."""
    from oracle import poly as op
    from sppark_b200 import poly
    f = op.FIELDS[field]
    p = f["p"]
    n = (1 << 22) + 3
    rng = np.random.default_rng(9)
    x = rng.integers(1, p, size=n, dtype=f["dtype"])          # non-zero memory words
    z, pt = _vals(field, 2, 5)
    zb, ptb = op.encode(field, [z]), op.encode(field, [pt])

    y = x.copy()
    poly.div_by_x_minus_z(y, zb)                              # [r, q...]
    r = op.decode(field, y[:1])[0]
    assert r == op.decode(field, poly.evaluate(x, zb))[0]
    pv = op.decode(field, poly.evaluate(x, ptb))[0]
    qv = op.decode(field, poly.evaluate(np.ascontiguousarray(y[1:]), ptb))[0]
    assert pv == (qv * (pt - z) + r) % p
    yr = x.copy()
    poly.div_by_x_minus_z(yr, zb, rotate=True)
    assert np.array_equal(yr[:-1], y[1:]) and yr[-1] == y[0]

    s = x.copy()
    poly.prefix_op(poly.ADD, s)
    # both memory formats are linear (plain words / Montgomery residues): sum the words themselves
    acc = sum(int(x[i:i + 65536].astype(object).sum()) for i in range(0, n, 65536))
    assert int(s[-1]) == acc % p

    m = x.copy()
    poly.prefix_op(poly.MULTIPLY, m)
    inv = x.copy()
    poly.batch_inverse(inv)
    poly.prefix_op(poly.MULTIPLY, inv)
    prod = m.copy()
    poly.batch_inverse(prod)
    assert np.array_equal(inv, prod)


def test_empty_and_errors():
    import torch
    from sppark_b200 import _lib, poly
    l = _lib.lib()
    s = torch.cuda.current_stream().cuda_stream
    buf = torch.zeros(4, dtype=torch.int64, device="cuda")
    for fn in (lambda: l.sppark_b200_prefix_op_dev(0, 0, buf.data_ptr(), buf.data_ptr(), 0, s),
               lambda: l.sppark_b200_batch_inverse_dev(0, buf.data_ptr(), buf.data_ptr(), 0, s),
               lambda: l.sppark_b200_evaluate_dev(0, buf.data_ptr(), buf.data_ptr(), 0, buf.data_ptr(), 4, s)):
        _lib.check(fn())
    # empty polynomial evaluates to zero
    buf.fill_(7)
    _lib.check(l.sppark_b200_evaluate_dev(0, buf.data_ptr(), buf.data_ptr(), 2, buf.data_ptr(), 0, s))
    torch.cuda.synchronize()
    assert buf[:2].tolist() == [0, 0]
    with pytest.raises(RuntimeError):
        _lib.check(l.sppark_b200_prefix_op_dev(99, 0, buf.data_ptr(), buf.data_ptr(), 4, s))
    with pytest.raises(RuntimeError):
        _lib.check(l.sppark_b200_prefix_op_dev(0, 2, buf.data_ptr(), buf.data_ptr(), 4, s))
    with pytest.raises(RuntimeError):
        _lib.check(l.sppark_b200_div_by_x_minus_z_dev(0, buf.data_ptr(), 4, None, 0, s))
    with pytest.raises(ValueError):
        poly.div_by_x_minus_z(np.zeros(4, dtype=np.uint64), np.zeros(2, dtype=np.uint64))


def test_tensor_arguments_stay_on_the_device():
    """torch tensors are used in place on torch's current stream (no host copies)"""
    import torch
    from oracle import poly as op
    from sppark_b200 import poly
    c = _vals("gl64", 3000, 8)
    t = torch.from_numpy(op.encode("gl64", c).view(np.int64)).cuda()
    poly.prefix_op(poly.ADD, t, field=0)
    torch.cuda.synchronize()
    assert np.array_equal(t.cpu().numpy().view(np.uint64), op.encode("gl64", op.prefix_op(op.GL64_P, "add", c)))
