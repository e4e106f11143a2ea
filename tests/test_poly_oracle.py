"""CPU: oracle/poly.py against the recordings of the reference's own polynomial kernels
(tests/golden/poly_*_ref_gpu.npz, generated on a GPU by tests/golden/make_golden.py gen_poly
through oracle/ref_poly.cu) -- this is what pins the oracle the GPU parity tests rely on."""
import hashlib
import os

import numpy as np
import pytest

from oracle import poly as op

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _sha(a):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), dtype=np.uint8)


@pytest.mark.parametrize("field", ["gl64", "bb31", "bls12_381_fr"])
def test_oracle_matches_reference_recordings(field):
    g = np.load(os.path.join(GOLDEN, f"poly_{field}_ref_gpu.npz"))
    p, big = op.FIELDS[field]["p"], int(g["big"])
    checked = 0
    for n in [int(v) for v in g["lens"]] + [big]:
        x = op.seeded_input(field, n, 4242) if n == big else g[f"in_{n}"]
        same = (lambda a, b: np.array_equal(_sha(a), b)) if n == big else np.array_equal
        c = op.decode(field, x)
        assert same(op.encode(field, op.prefix_op(p, "add", c)), g[f"add_{n}"]), (n, "add")
        cm = op.decode(field, g[f"mulin_{n}"]) if f"mulin_{n}" in g else c
        assert same(op.encode(field, op.prefix_op(p, "mul", cm)), g[f"mul_{n}"]), (n, "mul")
        for k, z in enumerate(op.decode(field, g[f"z_{n}"])):
            for rot in (0, 1):
                if f"div_{n}_{k}_{rot}" in g:
                    assert same(op.encode(field, op.div_by_x_minus_z(p, c, z, bool(rot))), g[f"div_{n}_{k}_{rot}"]), (n, k, rot)
                    checked += 1
        if f"eval_{n}" in g:
            xs = op.decode(field, g[f"x_{n}"])
            assert np.array_equal(op.encode(field, op.evaluate(p, c, xs)), g[f"eval_{n}"]), (n, "evaluate")
            checked += 1
    assert checked >= 8


def test_field_table_matches_the_c_oracle():
    """the moduli written out in oracle/poly.py are the ones oracle/ff.c derives its constants from"""
    from oracle import pyoracle as o
    for name, cname in (("bls12_381_fr", "bls12_381_fr"), ("pallas_fr", "vesta_fp"), ("vesta_fr", "pallas_fp"),
                        ("bn254_fr", "bn254_fr"), ("bls12_377_fr", "bls12_377_fr")):
        assert op.FIELDS[name]["p"] == o.ff_consts(cname)["p"], name


def test_encode_decode_and_identities():
    for field in op.FIELDS:
        p = op.FIELDS[field]["p"]
        vals = [0, 1, 2, p - 1, p // 3]
        assert op.decode(field, op.encode(field, vals)) == vals
        c = [5, 0, 7, p - 2, 11, 13]
        for z in (0, 1, 9, p - 1):
            b = op.div_by_x_minus_z(p, c, z)
            assert b[0] == op.evaluate(p, c, [z])[0]                       # remainder = p(z)
            x = 12345
            assert op.evaluate(p, c, [x])[0] == (op.evaluate(p, b[1:], [x])[0] * (x - z) + b[0]) % p
            assert op.div_by_x_minus_z(p, c, z, rotate=True) == b[1:] + b[:1]
        inv = op.batch_inversion(p, c)
        assert [a * b % p for a, b in zip(c, inv)] == [1, 0, 1, 1, 1, 1]


def test_seeded_input_is_a_fixed_function_of_the_seed():
    a = op.seeded_input("gl64", 4, 4242)
    assert a.tolist() == op.seeded_input("gl64", 4, 4242).tolist()
    for field in op.FIELDS:
        x = op.seeded_input(field, 100, 1)
        assert all(v < op.FIELDS[field]["p"] for v in op.decode(field, x))
        assert np.array_equal(op.encode(field, op.decode(field, x)), x)
