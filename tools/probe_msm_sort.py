"""GPU probe of the MSM's bucket sort: the `sort` phase and the whole device-resident BLS12-381 G1
MSM, for this tree's library and (optionally) a second build such as the parent commit's, loaded
side by side in one process and alternated round by round on the same card and the same buffers.

Sizes 2^22, 2^24, 2^26 (2^16 distinct points, replicated); scalars uniform below 2^254 (as bench.py
draws them), all equal, or two-valued.  Each round times, per build, one profiled call (phase
split from the library's own CUDA events; this tree's build also reports the sort's sub-phases)
and one unprofiled call (CUDA events around the call).  Prints median [min, max] per case with
the GPU name, power limit and SM clock, checks that both builds give the same group element, and
writes probe_msm_sort.json into --out.

    python tools/probe_msm_sort.py --out DIR [--base path/to/libsppark_b200.so] [--rounds 5]
                                   [--sizes 22,24,26] [--kinds uniform,equal,two_valued]
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
from sppark_b200 import _lib  # noqa: E402

P_BLS = 0x1a0111ea397fe69a4b1ba7b6434bacd764774b84f38512bf6730d2a0f6b0f6241eabfffeb153ffffb9feffffffffaaab
R_BLS = 0x73eda753299d7d483339d80809a1d80553bda402fffe5bfeffffffff00000001
M_DISTINCT = 1 << 16


def load(path):
    l = C.CDLL(path)
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


def scalars(kind, n, seed):
    if kind == "uniform":
        rng = np.random.default_rng(seed)
        sc = np.empty((n, 4), dtype=np.uint64)
        for s in range(0, n, 1 << 22):
            e = min(n, s + (1 << 22))
            sc[s:e] = rng.integers(0, 2**64, size=(e - s, 4), dtype=np.uint64)
        sc[:, 3] >>= np.uint64(2)
    else:
        vals = [R_BLS - 1] if kind == "equal" else [R_BLS - 5, 3]
        rows = np.array([[(v >> (64 * k)) & (2**64 - 1) for k in range(4)] for v in vals], dtype=np.uint64)
        sc = rows[np.arange(n) % len(vals)]
    return torch.from_numpy(np.ascontiguousarray(sc).view(np.int64)).cuda()


def same_point(a, b):
    """Jacobian (Montgomery limbs) equality by cross-multiplication: X1 Z2^2 = X2 Z1^2, Y1 Z2^3 = Y2 Z1^3"""
    def ints(r):
        return [sum(int(r[6 * c + k]) << (64 * k) for k in range(6)) for c in range(3)]
    (x1, y1, z1), (x2, y2, z2) = ints(a), ints(b)
    if z1 == 0 or z2 == 0:
        return z1 == z2
    return (x1 * z2 * z2 - x2 * z1 * z1) % P_BLS == 0 and (y1 * z2 ** 3 - y2 * z1 ** 3) % P_BLS == 0


def run(l, d_pts, d_sc, n, stream, profiled):
    out = np.zeros(18, dtype=np.uint64)
    l.sppark_b200_profile_enable(int(profiled))
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    check(l.sppark_b200_msm_dev(0, out.ctypes.data, d_pts.data_ptr(), n, d_sc.data_ptr(), stream))
    e1.record()
    e1.synchronize()
    phases = {}
    if profiled:
        names, ms = (C.c_char_p * 16)(), (C.c_float * 16)()
        for i in range(l.sppark_b200_profile_read(names, ms, 16)):
            phases[names[i].decode()] = phases.get(names[i].decode(), 0.0) + float(ms[i])
        l.sppark_b200_profile_enable(0)
    return e0.elapsed_time(e1), phases, out


def summary(xs):
    xs = sorted(xs)
    return {"median": xs[len(xs) // 2], "min": xs[0], "max": xs[-1], "n": len(xs)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--base", default=os.environ.get("SPPARK_B200_LIB"), help="a second build to alternate with")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--sizes", default="22,24,26")
    ap.add_argument("--kinds", default="uniform,equal,two_valued")
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    os.environ["SPPARK_B200_MSM_SORT_PROFILE"] = "1"           # sub-phases of the new sort; older builds ignore it
    new_path = os.path.join(ROOT, "sppark_b200", "libsppark_b200.so")
    builds = {"new": load(new_path)}
    if args.base and os.path.abspath(args.base) != os.path.abspath(new_path):
        builds["base"] = load(args.base)
    torch.cuda.init()
    stream = torch.cuda.current_stream().cuda_stream
    base_pts = torch.empty((M_DISTINCT, 12), dtype=torch.int64, device="cuda")
    check(builds["new"].sppark_b200_generate_points_dev(0, base_pts.data_ptr(), M_DISTINCT, stream))
    info = card()
    print(json.dumps({"gpu": info, "builds": {k: (new_path if k == "new" else args.base) for k in builds}}), flush=True)
    results = []
    for lg in [int(s) for s in args.sizes.split(",")]:
        n = 1 << lg
        d_pts = base_pts.repeat(n // M_DISTINCT, 1).contiguous()
        for kind in args.kinds.split(","):
            d_sc = scalars(kind, n, lg)
            samples = {k: {"total": [], "phases": {}} for k in builds}
            outs = {}
            for k, l in builds.items():                         # warm-up: modules, memory pool
                run(l, d_pts, d_sc, n, stream, False)
            for r in range(args.rounds):
                order = list(builds) if r % 2 == 0 else list(builds)[::-1]
                for k in order:
                    _, ph, _ = run(builds[k], d_pts, d_sc, n, stream, True)
                    t, _, outs[k] = run(builds[k], d_pts, d_sc, n, stream, False)
                    samples[k]["total"].append(t)
                    ph["sort_total"] = sum(v for p, v in ph.items() if p.startswith("sort"))
                    for p, v in ph.items():
                        samples[k]["phases"].setdefault(p, []).append(v)
            row = {"lg": lg, "kind": kind, "clock": card().get("clocks.sm")}
            for k in builds:
                row[k] = {"total_ms": summary(samples[k]["total"]),
                          "phases_ms": {p: summary(v) for p, v in samples[k]["phases"].items()}}
            if "base" in builds:
                row["same_result"] = same_point(outs["new"], outs["base"])
            results.append(row)
            for k in builds:
                t, s = row[k]["total_ms"], row[k]["phases_ms"]["sort_total"]
                subs = " ".join(f"{p}={v['median']:.2f}" for p, v in row[k]["phases_ms"].items()
                                if p.startswith("sort") and p != "sort_total")
                print(f"2^{lg} {kind:10s} {k:4s}  msm {t['median']:8.2f} [{t['min']:.2f}, {t['max']:.2f}] ms   "
                      f"sort {s['median']:7.2f} [{s['min']:.2f}, {s['max']:.2f}] ms   ({subs})", flush=True)
            if "base" in builds:
                print(f"2^{lg} {kind:10s} same group element: {row['same_result']}   SM clock {row['clock']} MHz", flush=True)
            del d_sc
        del d_pts
        torch.cuda.empty_cache()
    with open(os.path.join(args.out, "probe_msm_sort.json"), "w") as f:
        json.dump({"gpu": info, "results": results}, f, indent=1)


if __name__ == "__main__":
    main()
