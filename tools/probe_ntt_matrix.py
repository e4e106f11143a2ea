"""GPU probe of the NTT and LDE down the columns of a row-major (2^lg, width) matrix.  For each shape
and operation it times, alternating them in rounds:
  (a) matrix:    the matrix entry (sppark_b200_ntt_matrix_dev / sppark_b200_lde_matrix_dev);
  (b) transpose: torch transpose -> ntt_batch_dev / lde_batch_dev -> transpose back, what a caller
                 does without the matrix entries;
  (c) batch:     ntt_batch_dev / lde_batch_dev alone on column-contiguous data (a floor).
Then the candidate tile shapes behind the policy: the matrix entry with the digits of the transform
forced through SPPARK_B200_NTT_SPLIT (two passes of 2^12 rows and 4-column tiles against three passes
of 2^8 rows and 16-column tiles at 2^24 x 16).  Every figure is the median and [min, max] of
CUDA-event samples after warm-up.  GB/s is the algorithmic traffic over the median: 2 x matrix bytes
per pass of the transform (for an LDE: the inverse transform's passes on the input, the spread's
read of the input and write of the output, the forward transform's passes on the output), against
the H100's 3.35 TB/s.  The card name and power limit are read in the same run.  Prints one line per
case and writes probe_ntt_matrix.json into --out.

    python tools/probe_ntt_matrix.py --out DIR [--rounds 5] [--per-round 3] [--quick]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from sppark_b200 import _lib, ntt  # noqa: E402

GL_P = 2**64 - 2**32 + 1
BB_P = 0x78000001
FIELDS = {"gl64": (ntt.GL64, 8), "bb31": (ntt.BB31, 4)}
HBM = 3.35e12
SHAPES = [(20, 8), (20, 64), (20, 256), (22, 64), (24, 16)]
CANDIDATES = {(24, 16): ["12,12", "8,8,8"]}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in q.split(",")]
    except Exception as e:
        name, power = torch.cuda.get_device_name(0), f"unknown ({e})"
    return name, power


def matrix(field, lg, width):
    rng = np.random.default_rng(lg * 1000 + width)
    n = (1 << lg) * width
    if field == "gl64":
        a = rng.integers(0, GL_P, size=n, dtype=np.uint64).view(np.int64)
    else:
        a = rng.integers(0, BB_P, size=n, dtype=np.uint32).view(np.int32)
    return torch.from_numpy(a).cuda().view(1 << lg, width)


def passes(lg):
    return (lg + 11) // 12


def event_ms(fn, stream):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    fn()
    e1.record(stream)
    e1.synchronize()
    return e0.elapsed_time(e1)


def alternate(variants, stream, rounds, per_round, warm=2):
    names = list(variants)
    for name in names:
        for _ in range(warm):
            variants[name]()
    torch.cuda.synchronize()
    samples = {name: [] for name in names}
    for r in range(rounds):
        for name in names[r % len(names):] + names[:r % len(names)]:
            for _ in range(per_round):
                samples[name].append(event_ms(variants[name], stream))
    return {name: (float(np.median(v)), float(min(v)), float(max(v))) for name, v in samples.items()}


def with_split(fn, split):
    def run():
        if split:
            os.environ["SPPARK_B200_NTT_SPLIT"] = split
        try:
            fn()
        finally:
            os.environ.pop("SPPARK_B200_NTT_SPLIT", None)
    return run


def fmt(name, t, algo):
    med, lo, hi = t
    bw = algo / (med * 1e-3)
    return f"{name} {med:.3f} ms [{lo:.3f}, {hi:.3f}] ({bw / 1e9:.0f} GB/s, {100 * bw / HBM:.0f}%)"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--per-round", type=int, default=3)
    ap.add_argument("--quick", action="store_true", help="one shape (smoke run of the script)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("probe_ntt_matrix: no CUDA device (there is no CPU measurement)")
    os.makedirs(a.out, exist_ok=True)
    os.environ.pop("SPPARK_B200_NTT_SPLIT", None)
    name, power = card()
    print(f"{name}, power limit {power}; median [min, max] of {a.rounds} x {a.per_round} samples, "
          "variants alternated", flush=True)
    l = _lib.lib()
    st = torch.cuda.current_stream()
    s = st.cuda_stream
    res = {"gpu": name, "power_limit": power, "rounds": a.rounds, "per_round": a.per_round,
           "cases": [], "candidates": []}
    shapes = [(20, 64)] if a.quick else SHAPES
    for field, (fid, esz) in FIELDS.items():
        for lg, width in shapes:
            x = matrix(field, lg, width)
            xt = x.t().contiguous()                      # column-contiguous copy: the batch floor's input
            mbytes = (width << lg) * esz
            for op in ("ntt", "lde1", "lde2"):
                if op == "ntt":
                    algo = 2 * passes(lg) * mbytes

                    def va():
                        l.sppark_b200_ntt_matrix_dev(fid, x.data_ptr(), lg, width, ntt.NN, 0, 0, s)

                    def vb():
                        t = x.t().contiguous()
                        l.sppark_b200_ntt_batch_dev(fid, t.data_ptr(), lg, width, ntt.NN, 0, 0, s)
                        x.copy_(t.t())

                    def vc():
                        l.sppark_b200_ntt_batch_dev(fid, xt.data_ptr(), lg, width, ntt.NN, 0, 0, s)
                else:
                    lb = int(op[-1])
                    if (width << (lg + lb)) * esz > 8 << 30:
                        continue
                    obytes = mbytes << lb
                    algo = 2 * passes(lg) * mbytes + mbytes + obytes + 2 * passes(lg + lb) * obytes
                    out = torch.empty(((1 << lg) << lb) * width, dtype=x.dtype, device="cuda")
                    xc = x.clone()

                    def va(out=out, lb=lb, xc=xc):
                        l.sppark_b200_lde_matrix_dev(fid, out.data_ptr(), xc.data_ptr(), lg, lb, width, s)

                    def vb(out=out, lb=lb, xc=xc):
                        t = xc.t().contiguous()
                        tout = torch.empty_like(out)
                        l.sppark_b200_lde_batch_dev(fid, tout.data_ptr(), t.data_ptr(), lg, lb, width, s)
                        out.view((1 << lg) << lb, width).copy_(tout.view(width, (1 << lg) << lb).t())
                        xc.copy_(t.t())

                    def vc(out=out, lb=lb):
                        l.sppark_b200_lde_batch_dev(fid, out.data_ptr(), xt.data_ptr(), lg, lb, width, s)
                t = alternate({"matrix": va, "transpose": vb, "batch": vc}, st, a.rounds, a.per_round)
                res["cases"].append({"field": field, "lg": lg, "width": width, "op": op, "ms": t,
                                     "GBps": {k: algo / (v[0] * 1e-3) / 1e9 for k, v in t.items()}})
                print(f"{field} 2^{lg} x {width:3d} {op:4s}: " + "  ".join(fmt(k, v, algo) for k, v in t.items()),
                      flush=True)
                if op != "ntt":
                    del out, xc
            splits = [] if a.quick else CANDIDATES.get((lg, width), [])
            if splits:
                def vs():
                    l.sppark_b200_ntt_matrix_dev(fid, x.data_ptr(), lg, width, ntt.NN, 0, 0, s)
                t = alternate({sp: with_split(vs, sp) for sp in splits}, st, a.rounds, a.per_round)
                for sp in splits:
                    algo = 2 * len(sp.split(",")) * mbytes
                    res["candidates"].append({"field": field, "lg": lg, "width": width, "split": sp, "ms": t[sp],
                                              "GBps": algo / (t[sp][0] * 1e-3) / 1e9})
                    print(f"{field} 2^{lg} x {width:3d} ntt split {sp}: " + fmt(sp, t[sp], algo), flush=True)
            del x, xt
            torch.cuda.empty_cache()
    with open(os.path.join(a.out, "probe_ntt_matrix.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
