"""GPU probe: device-resident MSM on every curve for several builds of the library, loaded side by side
in one process and alternated round by round on the same card and the same buffers.

Cases: BLS12-381 G1 at 2^26 (the bench.py headline shape) and Pallas at 2^24, then BLS12-381 G1 and G2,
BN254 G1 / G2, BLS12-377 G1 / G2 and Vesta at 2^20; 2^16 distinct points (i+1)*G replicated,
uniform scalars below 2^254.  Each round times, per build, one profiled call (phase split from the
library's own CUDA events) and one unprofiled call (CUDA events around the call).  Prints median
[min, max] per case with the GPU name, power limit and SM clock, checks on the G1 curves that every
build returns the same group element, and writes probe_msm_curves.json into --out.  (The Jacobian
bytes may differ between calls: the sort places a bucket's entries in a run-dependent order.)

    python tools/probe_msm_curves.py --out DIR --builds new=sppark_b200/libsppark_b200.so,base=old.so
                                     [--rounds 5] [--cases bls12_381_g1,pallas,...]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from sppark_b200 import _lib, msm  # noqa: E402

M_DISTINCT = 1 << 16
MODULUS = {msm.BLS12_381_G1: 0x1a0111ea397fe69a4b1ba7b6434bacd764774b84f38512bf6730d2a0f6b0f6241eabfffeb153ffffb9feffffffffaaab,
           msm.BLS12_377_G1: 0x01ae3a4617c510eac63b05c06ca1493b1a22d9f300f5138f1ef3622fba094800170b5d44300000008508c00000000001,
           msm.BN254_G1: 0x30644e72e131a029b85045b68181585d97816a916871ca8d3c208c16d87cfd47,
           msm.PALLAS: 0x40000000000000000000000000000000224698fc094cf91b992d30ed00000001,
           msm.VESTA: 0x40000000000000000000000000000000224698fc0994a8dd8c46eb2100000001}
CASES = [("bls12_381_g1", msm.BLS12_381_G1, 26), ("pallas", msm.PALLAS, 24), ("bls12_381_g1", msm.BLS12_381_G1, 20),
         ("bls12_381_g2", msm.BLS12_381_G2, 20), ("bn254_g1", msm.BN254_G1, 20), ("bn254_g2", msm.BN254_G2, 20),
         ("bls12_377_g1", msm.BLS12_377_G1, 20), ("bls12_377_g2", msm.BLS12_377_G2, 20), ("vesta", msm.VESTA, 20)]


def load(path):
    l = C.CDLL(os.path.abspath(path))
    for name in ("sppark_b200_msm_dev", "sppark_b200_generate_points_dev"):
        getattr(l, name).restype = _lib.RustError
    l.sppark_b200_msm_dev.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]
    l.sppark_b200_generate_points_dev.argtypes = [C.c_int, C.c_void_p, C.c_size_t, C.c_void_p]
    l.sppark_b200_profile_enable.argtypes = [C.c_int]
    l.sppark_b200_profile_read.argtypes = [C.POINTER(C.c_char_p), C.POINTER(C.c_float), C.c_int]
    l.sppark_b200_profile_read.restype = C.c_int
    return l


def check(err):
    if err.code != 0:
        raise RuntimeError(f"sppark_b200 error {err.code}")


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        row = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), [s.strip() for s in row.split(",")]))
    except Exception as e:
        return {"name": torch.cuda.get_device_name(0), "error": str(e)}


def run(l, curve, nl, d_pts, d_sc, n, stream, profiled):
    out = np.zeros(3 * nl, dtype=np.uint64)
    l.sppark_b200_profile_enable(int(profiled))
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    check(l.sppark_b200_msm_dev(curve, out.ctypes.data, d_pts.data_ptr(), n, d_sc.data_ptr(), stream))
    e1.record()
    e1.synchronize()
    phases = {}
    if profiled:
        names, ms = (C.c_char_p * 16)(), (C.c_float * 16)()
        for i in range(l.sppark_b200_profile_read(names, ms, 16)):
            phases[names[i].decode()] = phases.get(names[i].decode(), 0.0) + float(ms[i])
        l.sppark_b200_profile_enable(0)
    return e0.elapsed_time(e1), phases, out


def same_point(curve, a, b):
    """Jacobian equality by cross-multiplication (holds in Montgomery form too); None for G2"""
    if curve not in MODULUS:
        return None
    p, nl = MODULUS[curve], msm._LIMBS[curve]

    def ints(r):
        return [sum(int(r[nl * c + k]) << (64 * k) for k in range(nl)) for c in range(3)]
    (x1, y1, z1), (x2, y2, z2) = ints(a), ints(b)
    if z1 == 0 or z2 == 0:
        return z1 == z2
    return (x1 * z2 * z2 - x2 * z1 * z1) % p == 0 and (y1 * z2 ** 3 - y2 * z1 ** 3) % p == 0


def summary(xs):
    xs = sorted(xs)
    return {"median": xs[len(xs) // 2], "min": xs[0], "max": xs[-1], "n": len(xs)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--builds", default="new=" + os.path.join(ROOT, "sppark_b200", "libsppark_b200.so"),
                    help="comma-separated name=path of the library builds to alternate")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--cases", default=",".join(c[0] for c in CASES))
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    paths = dict(b.split("=", 1) for b in args.builds.split(","))
    builds = {k: load(p) for k, p in paths.items()}
    torch.cuda.init()
    stream = torch.cuda.current_stream().cuda_stream
    info = card()
    print(json.dumps({"gpu": info, "builds": paths}), flush=True)
    first = next(iter(builds.values()))
    rng = np.random.default_rng(1)
    results = []
    for name, curve, lg in CASES:
        if name not in args.cases.split(",") and f"{name}@{lg}" not in args.cases.split(","):
            continue
        n, nl = 1 << lg, msm._LIMBS[curve]
        base = torch.empty((M_DISTINCT, 2 * nl), dtype=torch.int64, device="cuda")
        check(first.sppark_b200_generate_points_dev(curve, base.data_ptr(), M_DISTINCT, stream))
        d_pts = base.repeat(n // M_DISTINCT, 1).contiguous()
        sc = rng.integers(0, 2**64, size=(n, 4), dtype=np.uint64)
        sc[:, 3] >>= np.uint64(2)
        d_sc = torch.from_numpy(sc.view(np.int64)).cuda()
        samples = {k: {"total": [], "phases": {}} for k in builds}
        outs = {}
        for k, l in builds.items():                             # warm-up: modules, memory pool
            run(l, curve, nl, d_pts, d_sc, n, stream, False)
        for r in range(args.rounds):
            order = list(builds) if r % 2 == 0 else list(builds)[::-1]
            for k in order:
                _, ph, _ = run(builds[k], curve, nl, d_pts, d_sc, n, stream, True)
                t, _, outs[k] = run(builds[k], curve, nl, d_pts, d_sc, n, stream, False)
                samples[k]["total"].append(t)
                for p, v in ph.items():
                    samples[k]["phases"].setdefault(p, []).append(v)
        ref = outs[next(iter(outs))]
        same = [same_point(curve, ref, o) for o in outs.values()]
        row = {"case": name, "lg": lg, "clock": card().get("clocks.sm"),
               "same_group_element": None if None in same else all(same)}
        for k in builds:
            row[k] = {"total_ms": summary(samples[k]["total"]),
                      "phases_ms": {p: summary(v) for p, v in samples[k]["phases"].items()}}
        results.append(row)
        for k in builds:
            t, acc = row[k]["total_ms"], row[k]["phases_ms"].get("accumulate", {"median": 0, "min": 0, "max": 0})
            print(f"{name:13s} 2^{lg} {k:10s} msm {t['median']:8.2f} [{t['min']:.2f}, {t['max']:.2f}] ms   "
                  f"accumulate {acc['median']:8.2f} [{acc['min']:.2f}, {acc['max']:.2f}] ms", flush=True)
        print(f"{name:13s} 2^{lg} same group element: {row['same_group_element']}   SM clock {row['clock']}", flush=True)
        del d_pts, d_sc, base
        torch.cuda.empty_cache()
    with open(os.path.join(args.out, "probe_msm_curves.json"), "w") as f:
        json.dump({"gpu": info, "builds": paths, "results": results}, f, indent=1)


if __name__ == "__main__":
    main()
