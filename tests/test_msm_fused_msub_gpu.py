"""The fused a*b - c*d ladder (ff/mont.cuh msub_inline, called through msub_shared) with four
independent operands, bit-exact against Python integers on every field the self-test hook
covers.  BLS12-381 fr (top limb 0x73eda753) takes the two-ladder fallback, the others the fused
ladder."""
import random

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

FIELDS = [("bls12_381_fp", 0, 6), ("bls12_381_fr", 1, 4), ("pallas_fp", 2, 4), ("vesta_fp", 3, 4),
          ("bn254_fp", 4, 4), ("bn254_fr", 5, 4), ("bls12_377_fp", 6, 6), ("bls12_377_fr", 7, 4)]


def _limbs(x, n):
    return [(x >> (64 * i)) & 0xFFFFFFFFFFFFFFFF for i in range(n)]


def _int(row):
    return sum(int(v) << (64 * i) for i, v in enumerate(row))


def _quads(p, seed):
    rnd = random.Random(seed)
    corners = [0, 1, p - 1, p - 2]
    quads = [(a, b, c, d) for a in corners for b in corners for c in corners for d in corners]
    for _ in range(200):                            # d = 0: the subtrahend row is c_I * p
        quads.append((rnd.randrange(p), rnd.randrange(p), rnd.randrange(p), 0))
    for _ in range(200):                            # a*b = c*d mod p: zero result
        a, b, c = rnd.randrange(1, p), rnd.randrange(p), rnd.randrange(1, p)
        quads.append((a, b, c, a * b * pow(c, -1, p) % p))
        quads.append((a, b, b, a))
    quads += [tuple(rnd.randrange(p) for _ in range(4)) for _ in range(2000)]
    return quads


@pytest.mark.parametrize("name,fid,nl", FIELDS)
def test_msub_four_operands(oracle, name, fid, nl):
    from sppark_b200 import msm
    p = oracle.ff_consts(name)["p"]
    Rinv = pow(1 << (64 * nl), -1, p)
    quads = _quads(p, 1000 + fid)
    a = np.array([_limbs(v, nl) for q in quads for v in (q[0], q[2])], dtype=np.uint64)
    b = np.array([_limbs(v, nl) for q in quads for v in (q[1], q[3])], dtype=np.uint64)
    r = msm.selftest_field(fid, "msub4", a, b)
    assert r.shape == (len(quads), nl)
    for i, (x, y, z, w) in enumerate(quads):
        assert _int(r[i]) == (x * y - z * w) * Rinv % p, (name, i, hex(x), hex(y), hex(z), hex(w))
