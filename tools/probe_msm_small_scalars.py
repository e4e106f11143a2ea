"""GPU probe: MSM over small scalars.  Per curve, size and bit bound, three variants alternated in one
process on the same points and values: today's call with the values in 32-byte scalars ("full"), the
bounded call on the same 32-byte array ("bound32") and the bounded call on the compact array
("compact").  Device-resident and host-pinned paths, one preloaded-context case, and a
SPPARK_B200_MSM_WBITS sweep.  Prints median [min, max] ms per variant, the phases of the last profiled
call (profile_read) and the scratch-blob bytes of the chosen geometry.  Development tool, not the bench.

    python tools/probe_msm_small_scalars.py [--rounds R] [--lgs 20,22,24,26] [--out result.json]"""
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

CURVES = {"bls12_381": (msm.BLS12_381_G1, 6), "bn254": (msm.BN254_G1, 4)}
NBITS = [1, 8, 16, 32, 64, 128, 255]


def card():
    """name and power limit of the GPU, read (not changed) through nvidia-smi"""
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                       text=True, timeout=30).strip().splitlines()[torch.cuda.current_device()]
    except Exception as e:                                  # noqa: BLE001
        return f"{torch.cuda.get_device_name()} (power limit unknown: {e})"


def geometry(n, nbits, nl):
    """make_config(n, nbits) of msm_core.cuh in Python, and msm_t::begin's main scratch bytes:
    staging + sorted entries (12 B each), buckets and running-sum levels (XYZZ)"""
    best, best_cost = 4, None
    for c in range(4, 23):
        W = (nbits + c) // c
        cost = W * (1.11 * n + 5.5 * 2 ** (c - 1))
        e = nbits + 1 - (W - 1) * c
        if n >= 1 << 22 and e <= 10 and (n >> e) > 2048:
            cost += 1.25 * n
        if best_cost is None or cost < best_cost:
            best, best_cost = c, cost
    if os.environ.get("SPPARK_B200_MSM_WBITS"):
        best = int(os.environ["SPPARK_B200_MSM_WBITS"])
    W = (nbits + best) // best
    lg_l = max(best - 1 - 12, 0)
    items = W << (best - 1 - lg_l)
    xyzz = 4 * nl * 8
    return best, W, W * n * 12 + (W << (best - 1)) * xyzz + 3 * items * xyzz


def width(nbits):
    return next(sb for sb in (4, 8, 16, 32) if nbits <= 8 * sb)


def compact(sc4, sbytes):
    """(n, 4) uint64 rows -> the compact array of sbytes-byte scalars"""
    if sbytes == 32:
        return sc4
    if sbytes == 16:
        return np.ascontiguousarray(sc4[:, :2])
    if sbytes == 8:
        return np.ascontiguousarray(sc4[:, 0])
    return np.ascontiguousarray(sc4[:, 0]).astype(np.uint32)


def timed(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return 1e3 * (time.perf_counter() - t)


def stat(v):
    return {"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v))}


def run_case(cid, nl, n, nbits, path, rounds, d_pts, h_pts, ctx=None):
    rng = np.random.default_rng(nbits + n)
    sc4 = rng.integers(0, 2**64, size=(n, 4), dtype=np.uint64)
    for k in range(4):                                      # the same values below 2^nbits in every variant
        keep = nbits - 64 * k
        sc4[:, k] = 0 if keep <= 0 else sc4[:, k] & np.uint64((1 << keep) - 1 if keep < 64 else 2**64 - 1)
    sb = width(nbits)
    arrays = {"full": sc4, "bound32": sc4, "compact": compact(sc4, sb)}
    bound = {"full": None, "bound32": nbits, "compact": nbits}
    if path == "dev":
        dev = {k: torch.from_numpy(a.view(np.int32 if a.dtype == np.uint32 else np.int64)).cuda() for k, a in arrays.items()}
        call = {k: (lambda k=k: msm.msm_dev(cid, d_pts, dev[k], nbits=bound[k])) for k in arrays}
    else:
        pinned = {}
        for k, a in arrays.items():
            t = torch.empty(a.nbytes, dtype=torch.uint8).pin_memory()
            pinned[k] = t.numpy().view(a.dtype).reshape(a.shape)
            pinned[k][...] = a
        if ctx is not None:
            call = {k: (lambda k=k: ctx.invoke(pinned[k], nbits=bound[k])) for k in arrays}
        else:
            call = {k: (lambda k=k: msm.msm(cid, h_pts, pinned[k], nbits=bound[k])) for k in arrays}
    for k in arrays:                                        # warm-up
        call[k]()
    times = {k: [] for k in arrays}
    for _ in range(rounds):
        for k in arrays:
            times[k].append(timed(call[k]))
    phases = {}
    _lib.profile_enable(True)
    for k in arrays:
        call[k]()
        torch.cuda.synchronize()
        phases[k] = _lib.profile_read()
    _lib.profile_enable(False)
    c, W, blob = geometry(n, nbits, nl)
    c32, W32, blob32 = geometry(n, 255, nl)
    return {"n": n, "nbits": nbits, "path": path, "sbytes": sb,
            "wbits": c, "nwins": W, "scratch_bytes": blob, "wbits_full": c32, "nwins_full": W32, "scratch_bytes_full": blob32,
            "ms": {k: stat(v) for k, v in times.items()}, "phases": phases}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--lgs", default="20,22,24,26")
    ap.add_argument("--curves", default="bls12_381,bn254")
    ap.add_argument("--sweep", action="store_true", help="only the SPPARK_B200_MSM_WBITS sweep at 2^22")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    res = {"card": card(), "cases": []}
    print(res["card"], flush=True)
    lgs = [int(v) for v in args.lgs.split(",")]
    for name in args.curves.split(","):
        cid, nl = CURVES[name]
        for lg in ([22] if args.sweep else lgs):
            n = 1 << lg
            free, _ = torch.cuda.mem_get_info()
            if n * (16 * nl + 32) * 3 + geometry(n, 255, nl)[2] > free:
                print(f"{name} 2^{lg}: skipped, {free / 2**30:.1f} GiB free", flush=True)
                continue
            base = msm.generate_points_dev(cid, 1 << 16)
            d_pts = base.repeat(n >> 16, 1) if lg >= 16 else base[:n]
            h_t = torch.empty(d_pts.shape, dtype=torch.int64, pin_memory=True)
            h_t.copy_(d_pts)
            h_pts = h_t.numpy().view(np.uint64)
            sweeps = [(nb, c) for nb in (16, 64) for c in range(4, 23)] if args.sweep else [(nb, None) for nb in NBITS]
            for nbits, c in sweeps:
                if c is not None:
                    os.environ["SPPARK_B200_MSM_WBITS"] = str(c)
                for path in ("dev", "host"):
                    r = run_case(cid, nl, n, nbits, path, args.rounds, d_pts, h_pts)
                    r["curve"] = name
                    res["cases"].append(r)
                    ms = r["ms"]
                    print(f"{name} 2^{lg} nbits={nbits:3d} {path:4s} c={r['wbits']} W={r['nwins']} "
                          + " ".join(f"{k}={v['median']:.2f} [{v['min']:.2f},{v['max']:.2f}]" for k, v in ms.items()),
                          flush=True)
                os.environ.pop("SPPARK_B200_MSM_WBITS", None)
            if not args.sweep and name == "bls12_381" and lg == 22:
                ctx = msm.MsmContext(cid, h_pts)
                try:
                    for nbits in (16, 64):
                        r = run_case(cid, nl, n, nbits, "preloaded", args.rounds, d_pts, h_pts, ctx=ctx)
                        r["curve"] = name
                        res["cases"].append(r)
                        print(f"{name} 2^{lg} nbits={nbits:3d} preloaded "
                              + " ".join(f"{k}={v['median']:.2f}" for k, v in r["ms"].items()), flush=True)
                finally:
                    ctx.close()
            del d_pts, base
            torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
