"""oracle/poly.py -- TEST INFRASTRUCTURE ONLY (never imported by sppark_b200/).

CPU restatement, on Python integers, of what the reference's polynomial helpers and its batch
inversion compute (the reference code is cooperative CUDA; the arithmetic it performs is this):

  prefix_op            polynomial/prefix_op.cuh:17-45 (Add / Multiply) and :322-384 (host wrapper):
                       inclusive prefix over the field, out[i] = inp[0] (op) ... (op) inp[i]
  div_by_x_minus_z     polynomial/div_by_x_minus_z.cuh:112-154 (the comment that defines the
                       layout) and :445-486: synthetic division of c[0] + c[1] x + ... by (x - z);
                       rotate=False -> out[0] = remainder, out[1:] = quotient;
                       rotate=True  -> out[:-1] = quotient, out[-1] = remainder
  evaluate             polynomial/evaluate.cuh:304-414: ret[k] = sum_i coeffs[i] * x[k]^i
  batch_inversion      ff/batch_inversion.hpp:14-51: out[i] = 1 / inp[i], zero where inp[i] == 0

Pinned by tests/golden/poly_ref_gpu.npz: outputs of the reference's own kernels (oracle/ref_poly.cu
compiled from the reference sources, run on a GPU by tests/golden/make_golden.py gen_poly); the
reference itself holds no test or vector for these templates.  batch_inversion is header-only with
no entry point in the reference; it is pinned by its defining property (x * x^-1 == 1) only.

Memory formats (what the golden file and the C ABI carry):
  gl64   one canonical uint64                          (ff/gl64_t.cuh)
  bb31   one uint32 Montgomery residue, R = 2^32       (ff/mont32_t.cuh)
  fr256  8 x uint32 little-endian Montgomery residue, R = 2^256 (ff/mont_t.cuh)
"""
import numpy as np

GL64_P = 0xffffffff00000001
BB31_P = 0x78000001
BLS12_381_R = 0x73eda753299d7d483339d80809a1d80553bda402fffe5bfeffffffff00000001

PALLAS_P = 0x40000000000000000000000000000000224698fc094cf91b992d30ed00000001
VESTA_P = 0x40000000000000000000000000000000224698fc0994a8dd8c46eb2100000001
BN254_R = 0x30644e72e131a029b85045b68181585d2833e84879b9709143e1f593f0000001
BLS12_377_R = 0x12ab655e9a2ca55660b44d1e5c37b00159aa76fed00000010a11800000000001


def _wide(p):
    return dict(p=p, r=1 << 256, words=8, dtype=np.uint32)


# name -> modulus, Montgomery radix, 32-bit words per element; `id` = SPPARK_FIELD_* of the C ABI
FIELDS = {
    "gl64": dict(p=GL64_P, r=1, words=1, dtype=np.uint64, id=0),
    "bb31": dict(p=BB31_P, r=1 << 32, words=1, dtype=np.uint32, id=1),
    "bls12_381_fr": dict(_wide(BLS12_381_R), id=2),
    "pallas_fr": dict(_wide(VESTA_P), id=3),          # the scalar field of Pallas is Vesta's base field
    "vesta_fr": dict(_wide(PALLAS_P), id=4),
    "bn254_fr": dict(_wide(BN254_R), id=5),
    "bls12_377_fr": dict(_wide(BLS12_377_R), id=6),
}


def decode(field, a):
    """memory format -> list of true field values (Python ints)"""
    f = FIELDS[field]
    a = np.asarray(a)
    rinv = pow(f["r"], -1, f["p"])
    if f["words"] == 1:
        return [int(v) * rinv % f["p"] for v in a.reshape(-1)]
    a = a.reshape(-1, f["words"])
    out = []
    for row in a:
        v = 0
        for j in range(f["words"] - 1, -1, -1):
            v = (v << 32) | int(row[j])
        out.append(v * rinv % f["p"])
    return out


def encode(field, vals):
    """true values -> memory format"""
    f = FIELDS[field]
    if f["words"] == 1:
        return np.array([v * f["r"] % f["p"] for v in vals], dtype=f["dtype"])
    out = np.zeros((len(vals), f["words"]), dtype=np.uint32)
    for i, v in enumerate(vals):
        m = v * f["r"] % f["p"]
        for j in range(f["words"]):
            out[i, j] = (m >> (32 * j)) & 0xffffffff
    return out


def seeded_input(field, n, seed):
    """n memory-format elements from a seed, the same on every machine (numpy's PCG64 stream):
    lets a golden file keep digests of large outputs without the input arrays."""
    f = FIELDS[field]
    rng = np.random.default_rng(seed)
    if f["words"] == 1:
        return rng.integers(0, f["p"], size=n, dtype=f["dtype"])
    # any residue < p is a valid Montgomery word: clear the top bits, then fold the few >= p
    a = rng.integers(0, 1 << 32, size=(n, f["words"]), dtype=np.uint64).astype(np.uint32)
    a[:, -1] &= np.uint32((1 << (f["p"].bit_length() - 224 - 1)) - 1)
    return a


def prefix_op(p, op, inp):
    out, acc = [], None
    for v in inp:
        if acc is None:
            acc = v % p
        elif op == "add":
            acc = (acc + v) % p
        else:
            acc = acc * v % p
        out.append(acc)
    return out


def div_by_x_minus_z(p, c, z, rotate=False):
    n = len(c)
    b = [0] * n
    carry = 0
    for i in range(n - 1, -1, -1):          # b[i] = c[i] + z * b[i+1]
        carry = (c[i] + z * carry) % p
        b[i] = carry
    if rotate:
        return b[1:] + b[:1]
    return b


def evaluate(p, coeffs, xs):
    out = []
    for x in xs:
        acc = 0
        for c in reversed(coeffs):
            acc = (acc * x + c) % p
        out.append(acc)
    return out


def batch_inversion(p, inp):
    return [pow(v, -1, p) if v % p else 0 for v in inp]
