"""oracle/g2py.py -- TEST INFRASTRUCTURE ONLY (never imported by sppark_b200/).

G2 MSM of the reference's bn254 and bls12_377 builds (mult_pippenger_fp2_inf,
poc/msm-cuda/cuda/pippenger_inf.cu:8-13,36-47), restated on Python integers:

  Fp2 arithmetic        ff/alt_bn128-fp2.hpp (u^2 = -1), ff/bls12-377-fp2.hpp (u^2 = -5)
  point addition        the group law of y^2 = x^3 + b' in affine coordinates; what ec/jacobian_t.hpp:355-482
                        and ec/xyzz_t.hpp:117-200,352-429 compute projectively (a = 0: b' never appears)
  MSM                   msm/pippenger.hpp:192-214 `mult`: sum of double-and-add products

The C oracle (oracle/ec2.c) covers BLS12-381 G2 only; these two curves are small additions on top of
the same kernels, so a slow, obviously-right restatement is enough.  Pinned by
tests/golden/msm_g2_curves2_ref_gpu.npz: outputs of the reference's own CUDA templates for these
features (oracle/ref_msm_g2.cu built with FEATURE_BN254 / FEATURE_BLS12_377, run on a GPU by
tests/golden/make_golden.py g2_curves2).

Memory formats (what the C ABI carries): Fp = `nl` 64-bit little-endian limbs, Montgomery form
(R = 2^(64 nl)); Fp2 = (c0, c1); affine = (X, Y), all-zero = infinity; Jacobian = (X, Y, Z), Z = 0 = infinity.
"""
import math

import numpy as np

BN254_P = 0x30644e72e131a029b85045b68181585d97816a916871ca8d3c208c16d87cfd47
BN254_R = 0x30644e72e131a029b85045b68181585d2833e84879b9709143e1f593f0000001
BLS12_377_P = 0x01ae3a4617c510eac63b05c06ca1493b1a22d9f300f5138f1ef3622fba094800170b5d44300000008508c00000000001
BLS12_377_R = 0x12ab655e9a2ca55660b44d1e5c37b00159aa76fed00000010a11800000000001


class Curve:
    def __init__(self, name, cid, p, r, beta, nl, gen):
        self.name, self.id, self.p, self.r, self.beta, self.nl = name, cid, p, r, beta, nl
        self.R = 1 << (64 * nl)
        self.G = gen(self)

    # ---- Fp2 = Fp[u]/(u^2 + beta) ----
    def mul(self, a, b):
        p = self.p
        return ((a[0] * b[0] - self.beta * a[1] * b[1]) % p, (a[0] * b[1] + a[1] * b[0]) % p)

    def sub(self, a, b):
        return ((a[0] - b[0]) % self.p, (a[1] - b[1]) % self.p)

    def inv(self, a):
        d = pow(a[0] * a[0] + self.beta * a[1] * a[1], -1, self.p)
        return (a[0] * d % self.p, -a[1] * d % self.p)

    # ---- group law, affine; None = infinity ----
    def add(self, P, Q):
        if P is None or Q is None:
            return Q if P is None else P
        if P[0] == Q[0]:
            if self.sub((0, 0), P[1]) == Q[1]:
                return None
            lam = self.mul(self.mul((3, 0), self.mul(P[0], P[0])), self.inv(self.mul((2, 0), P[1])))
        else:
            lam = self.mul(self.sub(Q[1], P[1]), self.inv(self.sub(Q[0], P[0])))
        x = self.sub(self.sub(self.mul(lam, lam), P[0]), Q[0])
        return (x, self.sub(self.mul(lam, self.sub(P[0], x)), P[1]))

    def neg(self, P):
        return None if P is None else (P[0], self.sub((0, 0), P[1]))

    def smul(self, k, P):
        acc = None
        while k:
            if k & 1:
                acc = self.add(acc, P)
            P, k = self.add(P, P), k >> 1
        return acc

    def msm(self, points, scalars):
        acc = None
        for P, k in zip(points, scalars):
            acc = self.add(acc, self.smul(k, P))
        return acc

    # ---- memory formats ----
    def _fp(self, v):
        m = v * self.R % self.p
        return [(m >> (64 * i)) & 0xffffffffffffffff for i in range(self.nl)]

    def _unfp(self, limbs):
        v = 0
        for i in range(self.nl - 1, -1, -1):
            v = (v << 64) | int(limbs[i])
        return v * pow(self.R, -1, self.p) % self.p

    def encode_affine(self, points):
        """list of points (None = infinity) -> (n, 4 nl) uint64 rows"""
        out = np.zeros((len(points), 4 * self.nl), dtype=np.uint64)
        for i, P in enumerate(points):
            if P is not None:
                out[i] = self._fp(P[0][0]) + self._fp(P[0][1]) + self._fp(P[1][0]) + self._fp(P[1][1])
        return out

    def decode_affine(self, rows):
        nl, out = self.nl, []
        for row in np.asarray(rows).reshape(-1, 4 * nl):
            if not row.any():
                out.append(None)
                continue
            c = [self._unfp(row[k * nl:(k + 1) * nl]) for k in range(4)]
            out.append(((c[0], c[1]), (c[2], c[3])))
        return out

    def jacobian_to_affine(self, jac):
        nl = self.nl
        c = [self._unfp(np.asarray(jac)[k * nl:(k + 1) * nl]) for k in range(6)]
        X, Y, Z = (c[0], c[1]), (c[2], c[3]), (c[4], c[5])
        if Z == (0, 0):
            return None
        zi = self.inv(Z)
        zi2 = self.mul(zi, zi)
        return (self.mul(X, zi2), self.mul(Y, self.mul(zi2, zi)))


def _bn254_gen(c):
    # EIP-197 / arkworks bn254::g2 generator, y^2 = x^3 + 3/(9 + u)
    G = ((10857046999023057135944570762232829481370756359578518086990519993285655852781,
          11559732032986387107991004021392285783925812861821192530917403151452391805634),
         (8495653923123431417604973247489272438418190587263600148770280649306958101930,
          4082367875863433681332203403145435568316851327593401208105741076214120093531))
    b = c.mul((3, 0), c.inv((9, 1)))
    x3 = c.mul(c.mul(G[0], G[0]), G[0])
    assert c.mul(G[1], G[1]) == ((x3[0] + b[0]) % c.p, (x3[1] + b[1]) % c.p)
    return G


def _bls12_377_gen(c):
    # the same derivation as tools/gen_fields.py: P0 = (1 + u, 5 + 3u) lies on a sextic twist of order
    # n = p^2 + 1 - (t2 - 3 f2)/2, a multiple of r; G = (n / r) P0
    t = 0x8508c00000000001 + 1
    t2 = t * t - 2 * c.p
    f2 = math.isqrt((4 * c.p * c.p - t2 * t2) // 3)
    n = c.p * c.p + 1 - (t2 - 3 * f2) // 2
    assert n % c.r == 0
    return c.smul(n // c.r, ((1, 1), (5, 3)))


_CURVES = {}


def curve(name):
    if name not in _CURVES:
        if name == "bn254_g2":
            _CURVES[name] = Curve(name, 6, BN254_P, BN254_R, 1, 4, _bn254_gen)
        elif name == "bls12_377_g2":
            _CURVES[name] = Curve(name, 7, BLS12_377_P, BLS12_377_R, 5, 6, _bls12_377_gen)
        else:
            raise KeyError(name)
    return _CURVES[name]


def multiples(c, n):
    """[G, 2G, ..., nG]"""
    out, acc = [], None
    for _ in range(n):
        acc = c.add(acc, c.G)
        out.append(acc)
    return out


def scalars_to_rows(scalars):
    out = np.zeros((len(scalars), 4), dtype=np.uint64)
    for i, k in enumerate(scalars):
        for j in range(4):
            out[i, j] = (k >> (64 * j)) & 0xffffffffffffffff
    return out
