"""GPU probe (test infrastructure): which build of the REFERENCE's BabyBear / 256-bit NTT is
self-consistent on this GPU?  oracle/Makefile `ref-variants` builds, next to the sm_90a SASS
libraries, a PTX-only one (what the crate ships: rust/src/build.rs:54-57, JIT on the device) and
one with un-optimised device code.  For every library: the reference's own protocol
(poc/ntt-cuda/tests/ntt.rs: NN == RR, iNTT(NTT(x)) == x, NR -> RN round trip) and equality with
this repository's oracle."""
import ctypes as C
import os
import random
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import pyoracle as o  # noqa: E402

BB_P = 0x78000001
R_BLS = 0x73eda753299d7d483339d80809a1d80553bda402fffe5bfeffffffff00000001


class RE(C.Structure):
    _fields_ = [("code", C.c_int), ("message", C.c_void_p)]


def run(lib, x, lg, order, direction, typ=0):
    y = x.copy()
    e = lib.compute_ntt(0, y.ctypes.data, lg, order, direction, typ)
    assert e.code == 0, e.code
    return y


def main():
    # one process per field: the reference's parameter statics are STB_GNU_UNIQUE symbols, shared by
    # every library a process loads (tests/golden/make_golden.py explains)
    if len(sys.argv) < 2:
        import subprocess
        for f in ("bb31", "bls12_381_fr"):
            subprocess.check_call([sys.executable, os.path.abspath(__file__), f])
        return
    rnd = random.Random(5)
    for field, names in (("bb31", ["libref_ntt_bb31_gpu.so", "libref_ntt_bb31_gpu_ptx.so", "libref_ntt_bb31_gpu_O0.so"]),
                         ("bls12_381_fr", ["libref_ntt_bls12_381_gpu.so", "libref_ntt_bls12_381_gpu_ptx.so",
                                           "libref_ntt_bls12_381_gpu_O0.so"])):
        if field != sys.argv[1]:
            continue
        for name in names:
            path = o.ref_path(name)
            if not os.path.exists(path):
                print(name, "missing")
                continue
            lib = C.CDLL(path)
            lib.compute_ntt.restype = RE
            lib.compute_ntt.argtypes = [C.c_size_t, C.c_void_p, C.c_uint32, C.c_int, C.c_int, C.c_int]
            rows = []
            for lg in range(1, 13):
                n = 1 << lg
                if field == "bb31":
                    x = np.array([rnd.randrange(BB_P) for _ in range(n)], dtype=np.uint32)
                    want = o.ntt_bb31(x, o.NN) if lg <= 12 else None
                else:
                    x = np.array([o.int_to_limbs(rnd.randrange(R_BLS), 4) for _ in range(n)], dtype=np.uint64)
                    want = o.ntt_ff("bls12_381_fr", x, o.NN) if lg <= 10 else None
                nn = run(lib, x, lg, 0, 0)
                rr = run(lib, x, lg, 3, 0)
                back = run(lib, nn, lg, 0, 1)
                nr = run(lib, x, lg, 1, 0)
                rn = run(lib, nr, lg, 2, 1)
                cnn = run(lib, x, lg, 0, 0, 1)
                cback = run(lib, cnn, lg, 0, 1, 1)
                rows.append((lg, np.array_equal(nn, rr), np.array_equal(back, x), np.array_equal(rn, x),
                             np.array_equal(cback, x), None if want is None else np.array_equal(nn, want)))
            print(f"{name}:")
            print("   lg  NN==RR  iNTT(NTT)  NR->RN  coset-rt  ==oracle")
            for r in rows:
                print("   %2d  %-6s  %-9s  %-6s  %-8s  %s" % r)
            sys.stdout.flush()


if __name__ == "__main__":
    main()
