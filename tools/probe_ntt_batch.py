"""GPU probe of the batched NTT: one sppark_b200_ntt_batch_dev call against a loop of
sppark_b200_ntt_dev over the same rows, device-resident, every shape totalling 2^26 elements; then
the host-pointer entry sppark_b200_ntt_batch against a loop of sppark_b200_ntt, pinned and pageable.
Order NN, forward.  Every case is timed in several rounds with the order of its variants rotated
from round to round; it reports the median and the [min, max] of CUDA-event (device) or host-clock
(host entries, which synchronise) samples after warm-up.  `GB/s` is the algorithmic traffic of one pass,
2 * batch * 2^lg * sizeof(element), over the time.  Prints one line per case and writes
probe_ntt_batch.json into --out.

    python tools/probe_ntt_batch.py --out DIR [--rounds 7] [--per-round 3] [--quick]
"""
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
from sppark_b200 import _lib, ntt  # noqa: E402

GL_P = 2**64 - 2**32 + 1
BB_P = 0x78000001
TOTAL_LG = 26
FIELDS = {"gl64": (ntt.GL64, 8), "bb31": (ntt.BB31, 4), "bls12_381_fr": (ntt.BLS12_381_FR, 32)}
ENV = ("SPPARK_B200_NTT_WARP", "SPPARK_B200_NTT_BLOCK")


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in q.split(",")]
    except Exception as e:            # the name still comes from torch
        name, power = torch.cuda.get_device_name(0), f"unknown ({e})"
    return name, power


def device_data(field, batch, lg):
    rng = np.random.default_rng(lg)
    n = batch << lg
    if field == "gl64":
        return torch.from_numpy(rng.integers(0, GL_P, size=n, dtype=np.uint64).view(np.int64)).cuda()
    if field == "bb31":
        return torch.from_numpy(rng.integers(0, BB_P, size=n, dtype=np.uint32).view(np.int32)).cuda()
    # random residues below 2^254 < r(BLS12-381)
    a = rng.integers(0, 2**63, size=(n, 4), dtype=np.uint64)
    a[:, 3] >>= np.uint64(2)
    return torch.from_numpy(a.view(np.int64)).cuda()


def event_ms(fn, stream):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    fn()
    e1.record(stream)
    e1.synchronize()
    return e0.elapsed_time(e1)


def host_ms(fn, stream=None):
    t0 = time.perf_counter()
    fn()
    return (time.perf_counter() - t0) * 1e3


def alternate(variants, timer, stream, rounds, per_round, warm=2):
    """Times every variant in `rounds` rounds, `per_round` samples each, rotating the order of
    the variants from round to round so that clock and power drift fall on all of them alike.
    Returns {name: (median, min, max)} in ms."""
    names = list(variants)
    for name in names:
        for _ in range(warm):
            variants[name]()
    torch.cuda.synchronize()
    samples = {name: [] for name in names}
    for r in range(rounds):
        for name in names[r % len(names):] + names[:r % len(names)]:
            for _ in range(per_round):
                samples[name].append(timer(variants[name], stream))
    return {name: (float(np.median(v)), float(min(v)), float(max(v))) for name, v in samples.items()}


def with_env(fn, var):
    def run():
        for k in ENV:
            os.environ.pop(k, None)
        if var:
            os.environ[var] = "1"
        try:
            fn()
        finally:
            if var:
                os.environ.pop(var)
    return run


def fmt(name, t, algo):
    med, lo, hi = t
    return f"{name} {med:.3f} ms [{lo:.3f}, {hi:.3f}] ({algo / (med * 1e-3) / 1e9:.0f} GB/s)"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--per-round", type=int, default=3)
    ap.add_argument("--quick", action="store_true", help="fewer shapes (smoke run of the script)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("probe_ntt_batch: no CUDA device (there is no CPU measurement)")
    os.makedirs(a.out, exist_ok=True)
    name, power = card()
    print(f"{name}, power limit {power}; median [min, max] of {a.rounds} x {a.per_round} samples, "
          "variants alternated", flush=True)
    l = _lib.lib()
    st = torch.cuda.current_stream()
    s = st.cuda_stream
    results = {"gpu": name, "power_limit": power, "rounds": a.rounds, "per_round": a.per_round,
               "device": [], "host": []}

    # (field, lg, total lg): 2^26 elements per shape; rows of 2^3 also as a batch of 2^19 (the block
    # path with one row per tile), without the loop of 2^19 single calls
    shapes = [("gl64", lg, TOTAL_LG) for lg in (12, 16, 20, 24)] + [("bb31", lg, TOTAL_LG) for lg in (12, 16, 20, 24)] + \
             [("bls12_381_fr", lg, TOTAL_LG) for lg in (12, 16, 20)] + [("gl64", 3, 22), ("bb31", 3, 22)]
    if a.quick:
        shapes = [("gl64", 16, TOTAL_LG), ("bb31", 3, 22), ("bls12_381_fr", 12, TOTAL_LG)]
    for field, lg, total in shapes:
        fid, esz = FIELDS[field]
        batch = 1 << (total - lg)
        d = device_data(field, batch, lg)
        ptr, row = d.data_ptr(), esz << lg
        algo = 2 * batch * (1 << lg) * esz

        def loop():
            for b in range(batch):
                l.sppark_b200_ntt_dev(fid, ptr + b * row, lg, ntt.NN, 0, 0, s)

        def batched():
            l.sppark_b200_ntt_batch_dev(fid, ptr, lg, batch, ntt.NN, 0, 0, s)

        variants = {"batch": with_env(batched, None)}
        if batch <= 1 << 14:
            variants["loop"] = with_env(loop, None)
        if fid in (ntt.GL64, ntt.BB31):
            variants["batch_warp"] = with_env(batched, "SPPARK_B200_NTT_WARP")
            variants["batch_block"] = with_env(batched, "SPPARK_B200_NTT_BLOCK")
        t = alternate(variants, event_ms, st, a.rounds, a.per_round)
        rec = {"field": field, "lg": lg, "batch": batch, "ms": t,
               "GBps": {k: algo / (v[0] * 1e-3) / 1e9 for k, v in t.items()}}
        results["device"].append(rec)
        print(f"dev  {field:13s} 2^{lg:<2d} x {batch:6d}: " + "  ".join(fmt(k, v, algo) for k, v in t.items()),
              flush=True)
        del d
        torch.cuda.empty_cache()

    # host-pointer entries: gl64, 2^26 elements (512 MiB) as rows of 2^lg
    host_shapes = [20] if a.quick else [16, 20]
    rng = np.random.default_rng(1)
    src = rng.integers(0, GL_P, size=1 << TOTAL_LG, dtype=np.uint64)
    pinned = torch.empty(1 << TOTAL_LG, dtype=torch.int64).pin_memory()
    bufs = {"pinned": pinned.numpy().view(np.uint64), "pageable": np.empty(1 << TOTAL_LG, dtype=np.uint64)}
    algo = 2 * (8 << TOTAL_LG)
    for lg in host_shapes:
        batch = 1 << (TOTAL_LG - lg)
        for kind, buf in bufs.items():
            buf[:] = src
            p, row = buf.ctypes.data, 8 << lg

            def hloop():
                for b in range(batch):
                    _lib.check(l.sppark_b200_ntt(ntt.GL64, 0, p + b * row, lg, ntt.NN, 0, 0))

            def hbatch():
                _lib.check(l.sppark_b200_ntt_batch(ntt.GL64, 0, p, lg, batch, ntt.NN, 0, 0))

            t = alternate({"loop": hloop, "batch": hbatch}, host_ms, None, max(3, a.rounds // 2), 1, warm=1)
            results["host"].append({"field": "gl64", "lg": lg, "batch": batch, "memory": kind, "ms": t})
            print(f"host gl64 2^{lg} x {batch} {kind:8s}: " + "  ".join(fmt(k, v, algo) for k, v in t.items()),
                  flush=True)
    with open(os.path.join(a.out, "probe_ntt_batch.json"), "w") as f:
        json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
