"""GPU probe: a preloaded-point MSM context without a table against one with a precomputed
fixed-base table (MsmContext(..., precompute=K)), alternated in one process on the same points and
scalars.  Prints, per size: the invoke time (median [min, max] over the repetitions), the phases of
the last profiled invoke of each kind, the one-time context build time and the device bytes of the
points / table.  Development tool, not the bench.

    python tools/probe_msm_precomputed.py [--reps R] [--out result.json] [case ...]

A case is curve:lg:K, e.g. bls12_381:20:4; K = D takes the chooser's digit count for one bucket set,
K = max the largest K whose context and invoke fit the free device memory.  Without cases: the
table of DESIGN.md section 5a."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from sppark_b200 import _lib, msm  # noqa: E402
from oracle import pyoracle  # noqa: E402  (development tool: result comparison only)

CURVES = {"bls12_381": (msm.BLS12_381_G1, 96), "bn254": (msm.BN254_G1, 64), "pallas": (msm.PALLAS, 64),
          "bls12_381_g2": (msm.BLS12_381_G2, 192)}
DEFAULT = ([f"bls12_381:{lg}:{k}" for lg in (16, 18, 20, 22, 24) for k in ("4", "D")]
           + ["bls12_381:26:max", "bn254:20:D", "pallas:20:D", "bls12_381_g2:20:D"])


def card():
    """name and power limit of the GPU, read (not changed) through nvidia-smi"""
    try:
        q = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                    text=True, timeout=30).strip().splitlines()[torch.cuda.current_device()]
        return q
    except Exception as e:                                  # noqa: BLE001
        return f"{torch.cuda.get_device_name()} (power limit unknown: {e})"


def k_single_set(lg):
    """K = D: the smallest K for which the cost model chooses one bucket set (V = 1)"""
    best = None
    for c in range(4, 25):
        D = -(-256 // c)
        cost = 1.11 * D * (1 << lg) + 5.5 * 2 ** (c - 1)
        if best is None or cost < best[0]:
            best = (cost, D)
    return best[1]


def inputs(cid, lg):
    n = 1 << lg
    base = msm.generate_points_dev(cid, 1 << min(lg, 16))
    pts = torch.empty((n, base.shape[1]), dtype=torch.int64, pin_memory=True)
    pts.copy_(base.repeat(n // base.shape[0], 1))
    sc = torch.empty((n, 4), dtype=torch.int64, pin_memory=True)
    g = torch.Generator(device="cuda").manual_seed(lg)
    s = torch.randint(-2**63, 2**63 - 1, (n, 4), dtype=torch.int64, device="cuda", generator=g)
    s[:, 3] &= (1 << 62) - 1                                # below 2^254
    sc.copy_(s)
    torch.cuda.synchronize()
    del base, s
    return pts.numpy().view(np.uint64), sc.numpy().view(np.uint64)


def timed_invoke(ctx, sc):
    _lib.profile_enable(True)
    t0 = time.perf_counter()
    out = ctx.invoke(sc)
    ms = (time.perf_counter() - t0) * 1e3
    torch.cuda.synchronize()
    phases = _lib.profile_read()
    _lib.profile_enable(False)
    return ms, out, phases


def affine(curve, jac):
    """Jacobian limbs -> affine (the representative of a point varies from call to call)"""
    return pyoracle.g2_jac_to_affine(jac) if curve == "bls12_381_g2" else pyoracle.jac_to_affine(curve, jac)


def stats(v):
    v = sorted(v)
    return {"median": v[len(v) // 2], "min": v[0], "max": v[-1]}


def run_case(case, reps):
    curve, lg, k = case.split(":")
    lg = int(lg)
    cid, row = CURVES[curve]
    pts, sc = inputs(cid, lg)
    t0 = time.perf_counter()
    plain = msm.MsmContext(cid, pts)
    plain_build = (time.perf_counter() - t0) * 1e3
    ks = [k_single_set(lg)] if k == "D" else list(range(k_single_set(lg), 1, -1)) if k == "max" else [int(k)]
    table, err = None, None
    for K in ks:
        try:
            t0 = time.perf_counter()
            table = msm.MsmContext(cid, pts, precompute=K)
            table_build = (time.perf_counter() - t0) * 1e3
            timed_invoke(table, sc)                         # warm-up; fails here when the scratch does not fit
            break
        except _lib.SpparkError as e:
            err = str(e)
            if table is not None:
                table.close()
            table = None
            torch.cuda.empty_cache()
    if table is None:
        plain.close()
        return {"case": case, "error": err}
    timed_invoke(plain, sc)
    tp, tt = [], []
    for _ in range(reps):                                   # alternated
        ms, out_p, ph_p = timed_invoke(plain, sc)
        tp.append(ms)
        ms, out_t, ph_t = timed_invoke(table, sc)
        tt.append(ms)
    os.environ["SPPARK_B200_MSM_DEBUG"] = "1"
    r, w = os.pipe()
    saved = os.dup(2)
    os.dup2(w, 2)
    try:
        table.invoke(sc)
    finally:
        os.dup2(saved, 2)
        os.close(w)
        os.environ.pop("SPPARK_B200_MSM_DEBUG")
    line = os.read(r, 1 << 16).decode().strip().splitlines()[-1]
    os.close(r)
    geo = dict(kv.split("=") for kv in line.split() if "=" in kv)
    copies = int(geo["copies"])
    res = {"case": case, "curve": curve, "lg": lg, "K": K, "wbits": int(geo["wbits"]), "sets": int(geo["sets"]),
           "digits": int(geo["digits"]), "copies": copies,
           "same_point": bool(np.array_equal(affine(curve, out_p), affine(curve, out_t))),
           "plain_ms": stats(tp), "table_ms": stats(tt), "plain_phases": ph_p, "table_phases": ph_t,
           "plain_build_ms": plain_build, "table_build_ms": table_build,
           "points_bytes": (1 << lg) * row, "table_bytes": copies * (1 << lg) * row}
    plain.close()
    table.close()
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out")
    ap.add_argument("cases", nargs="*")
    a = ap.parse_args()
    gpu = card()
    print(f"# {gpu}", flush=True)
    results = []
    for case in a.cases or DEFAULT:
        res = run_case(case, a.reps)
        results.append(res)
        if "error" in res:
            print(f"{case}: {res['error']}", flush=True)
            continue
        p, t = res["plain_ms"], res["table_ms"]
        print(f"{case:>18} K={res['K']:<2} c={res['wbits']:<2} V={res['sets']:<2} D={res['digits']:<2} copies={res['copies']:<2}"
              f" plain {p['median']:8.2f} [{p['min']:.2f}, {p['max']:.2f}] ms  table {t['median']:8.2f}"
              f" [{t['min']:.2f}, {t['max']:.2f}] ms  ({100 * (t['median'] / p['median'] - 1):+.1f} %)"
              f"  build {res['table_build_ms']:.0f} ms (plain {res['plain_build_ms']:.0f})"
              f"  table {res['table_bytes'] / 2**30:.2f} GiB  same={res['same_point']}", flush=True)
        fmt = lambda ph: " ".join(f"{k}={v:.2f}" for k, v in ph)  # noqa: E731
        print(f"{'':>18} phases plain: {fmt(res['plain_phases'])}", flush=True)
        print(f"{'':>18} phases table: {fmt(res['table_phases'])}", flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump({"gpu": gpu, "results": results}, f, indent=1)


if __name__ == "__main__":
    main()
