"""GPU probe: the batched MSM entries against a loop of single calls on the same context and inputs,
alternated in one process: MsmContext.invoke_batch against B calls of invoke (plain context and a
precomputed one of K = 4 copies), msm_dev_batch against B calls of msm_dev.  Prints, per shape: both
times (median [min, max] over the repetitions, host clock around calls that end in a synchronise), the
group size the entry chose, and whether every vector's result is the same point both ways; then the
phases (profile_read) of one batched and one single call of a small shape.  Development tool, not the
bench.

    python tools/probe_msm_batch.py [--reps R] [--out result.json] [case ...]

A case is curve:lg:B:mode with mode plain, k4 or dev, e.g. bls12_381:16:64:plain.  Without cases:
the table of DESIGN.md section 5d."""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from sppark_b200 import _lib, msm  # noqa: E402
from probe_msm_precomputed import affine, card, stats  # noqa: E402  (oracle: result comparison only)

CURVES = {"bls12_381": msm.BLS12_381_G1, "bn254": msm.BN254_G1, "bls12_381_g2": msm.BLS12_381_G2}
DEFAULT = ([f"{c}:{lg}:{B}:{m}" for c in ("bls12_381", "bn254") for m in ("plain", "k4", "dev")
            for lg in (12, 14, 16, 18, 20) for B in (1, 4, 16, 64)]
           + [f"bls12_381_g2:16:{B}:{m}" for m in ("plain", "k4", "dev") for B in (1, 4, 16, 64)])


class Inputs:
    """points of one curve and size (device and host) and B vectors of scalars below 2^254"""
    def __init__(self, cid, lg, B):
        n = 1 << lg
        base = msm.generate_points_dev(cid, 1 << min(lg, 16))
        self.d_pts = base.repeat(n // base.shape[0], 1).contiguous()
        g = torch.Generator(device="cuda").manual_seed(lg * 100 + B)
        self.d_sc = torch.randint(-2**63, 2**63 - 1, (B, n, 4), dtype=torch.int64, device="cuda", generator=g)
        self.d_sc[:, :, 3] &= (1 << 62) - 1
        self.pts = self.d_pts.cpu().numpy().view(np.uint64)
        self.sc = torch.empty((B, n, 4), dtype=torch.int64, pin_memory=True)
        self.sc.copy_(self.d_sc)
        self.sc = self.sc.numpy().view(np.uint64)
        torch.cuda.synchronize()


def groups_of(call):
    """the vectors per group of one call, from its SPPARK_B200_MSM_DEBUG lines"""
    os.environ["SPPARK_B200_MSM_DEBUG"] = "1"
    r, w = os.pipe()
    saved = os.dup(2)
    os.dup2(w, 2)
    try:
        call()
    finally:
        os.dup2(saved, 2)
        os.close(w)
        os.close(saved)
        os.environ.pop("SPPARK_B200_MSM_DEBUG")
    text = os.read(r, 1 << 20).decode()
    os.close(r)
    return [int(kv.split("=")[1]) for ln in text.splitlines() for kv in ln.split() if kv.startswith("vecs=")]


def run_case(case, reps, cache):
    curve, lg, B, mode = case.split(":")
    lg, B = int(lg), int(B)
    cid = CURVES[curve]
    key = (curve, lg, B)
    if cache.get("key") != key:
        cache.clear()
        torch.cuda.empty_cache()
        cache["key"], cache["inp"] = key, Inputs(cid, lg, B)
    inp = cache["inp"]
    if mode == "dev":
        batch = lambda: msm.msm_dev_batch(cid, inp.d_pts, inp.d_sc)                            # noqa: E731
        loop = lambda: np.stack([msm.msm_dev(cid, inp.d_pts, inp.d_sc[b]) for b in range(B)])  # noqa: E731
        ctx = None
    else:
        ctx = msm.MsmContext(cid, inp.pts, precompute=4 if mode == "k4" else None)
        batch = lambda: ctx.invoke_batch(inp.sc)                                               # noqa: E731
        loop = lambda: np.stack([ctx.invoke(inp.sc[b]) for b in range(B)])                   # noqa: E731
    batch(), loop()                                                                             # warm-up
    tb, tl = [], []
    for _ in range(reps):                                                                       # alternated
        t0 = time.perf_counter()
        ob = batch()
        tb.append((time.perf_counter() - t0) * 1e3)
        t0 = time.perf_counter()
        ol = loop()
        tl.append((time.perf_counter() - t0) * 1e3)
    same = all(np.array_equal(affine(curve, ob[b]), affine(curve, ol[b])) for b in range(B))
    res = {"case": case, "curve": curve, "lg": lg, "B": B, "mode": mode, "groups": groups_of(batch),
           "batch_ms": stats(tb), "loop_ms": stats(tl), "same_point": same}
    if ctx is not None:
        ctx.close()
    return res


def phases(reps):
    """profile_read of one batched call and of one single call: BLS12-381 G1, 2^12 points, 16 vectors"""
    cid = CURVES["bls12_381"]
    inp = Inputs(cid, 12, 16)
    ctx = msm.MsmContext(cid, inp.pts)
    out = {}
    for name, call in (("batch16", lambda: ctx.invoke_batch(inp.sc)), ("single", lambda: ctx.invoke(inp.sc[0]))):
        for _ in range(reps):
            call()
        _lib.profile_enable(True)
        call()
        torch.cuda.synchronize()
        out[name] = _lib.profile_read()
        _lib.profile_enable(False)
    ctx.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out")
    ap.add_argument("cases", nargs="*")
    a = ap.parse_args()
    gpu = card()
    print(f"# {gpu}", flush=True)
    results, cache = [], {}
    for case in a.cases or DEFAULT:
        res = run_case(case, a.reps, cache)
        results.append(res)
        b, l = res["batch_ms"], res["loop_ms"]
        print(f"{case:>28} groups={res['groups']}  batch {b['median']:9.2f} [{b['min']:.2f}, {b['max']:.2f}] ms"
              f"  loop {l['median']:9.2f} [{l['min']:.2f}, {l['max']:.2f}] ms  x{l['median'] / b['median']:.2f}"
              f"  same={res['same_point']}", flush=True)
    cache.clear()
    ph = phases(a.reps)
    for name, p in ph.items():
        print(f"# phases {name}: " + " ".join(f"{k}={v:.3f}" for k, v in p), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump({"gpu": gpu, "results": results, "phases": ph}, f, indent=1)


if __name__ == "__main__":
    main()
