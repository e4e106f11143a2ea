"""Which form of a*b - c*d each field's constants select (ff/mont.cuh msub_inline): the fused
one-reduction ladder needs 3p < 2^(32N); larger moduli fall back to two product ladders.  Every
G1 base field must take the fused form, since it is the subtraction of the MSM's mixed add."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FF = os.path.join(ROOT, "sppark_b200", "csrc", "ff")

FUSED = {"bls12_381_fp", "pallas_fp", "vesta_fp", "bn254_fp", "bls12_377_fp", "bn254_fr", "bls12_377_fr"}
FALLBACK = {"bls12_381_fr"}


def _fields():
    src = open(os.path.join(FF, "fields.cuh")).read()
    out = {}
    for m in re.finditer(r"struct (\w+)_params \{\s*static constexpr int N = (\d+);.*?"
                         r"P\(int i\) \{ constexpr uint32_t t\[\d+\] = \{([^}]*)\}", src, re.S):
        limbs = [int(x.strip().rstrip("u"), 16) for x in m.group(3).split(",")]
        assert len(limbs) == int(m.group(2))
        out[m.group(1)] = limbs
    return out


def _fallback_threshold():
    src = open(os.path.join(FF, "mont.cuh")).read()
    m = re.search(r"mont_t msub_inline\(.*?\)\s*\{\s*if constexpr \(C::P\(N - 1\) >= (0x[0-9a-fA-F]+)u\)", src, re.S)
    assert m, "msub_inline's branch condition not found"
    return int(m.group(1), 16)


def test_msub_branch_per_field():
    fields = _fields()
    assert set(fields) == FUSED | FALLBACK
    threshold = _fallback_threshold()
    for name, limbs in fields.items():
        n = len(limbs)
        p = sum(v << (32 * i) for i, v in enumerate(limbs))
        fused = limbs[n - 1] < threshold
        if fused:                                   # the rule only admits moduli the ladder's bound holds for
            assert 3 * p < 1 << (32 * n), name
        assert fused == (name in FUSED), (name, hex(limbs[n - 1]))
