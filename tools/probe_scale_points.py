"""GPU probe: scalar multiplication of point arrays (sppark_b200_scale_points[_dev], DESIGN.md section 5e).

  device entry  BLS12-381 G1, BN254 G1, Pallas, BLS12-381 G2 at 2^16 .. 2^22 points, 255-bit (32-byte)
                and 64-bit (8-byte) scalars: CUDA events around one call, the cases alternated round by
                round, median [min, max] over the rounds
  host entry    BLS12-381 G1 at 2^20, pinned and pageable rows: host clock around the call (it ends in a
                synchronise)
  ladder share  the ladder kernel's time from torch.profiler (a run of its own, BLS12-381 G1, 2^20,
                255-bit scalars) against the IMAD.WIDE bound of the product count in DESIGN.md section 5e

Prints the card's name and power limit first.  Development tool, not the bench.

    python tools/probe_scale_points.py [--rounds R] [--lgs 16,18,20,22] [--curves a,b] [--device-only]
                                       [--out result.json]"""
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
from sppark_b200 import msm  # noqa: E402
from probe_msm_precomputed import card, stats  # noqa: E402

CURVES = {"bls12_381": msm.BLS12_381_G1, "bn254": msm.BN254_G1, "pallas": msm.PALLAS,
          "bls12_381_g2": msm.BLS12_381_G2}
# IMAD.WIDE per product for BLS12-381 G1, w = 5, 255-bit scalars: 255 doublings x 2250, ~50 additions
# x 3756, the table 15 madd x 2604 (DESIGN.md section 5e); 0.92 warp-instructions per SM per clock (section 5)
IMAD_PER_PRODUCT = 255 * 2250 + 50 * 3756 + 15 * 2604
IMAD_RATE_PER_SM_CLK = 0.92 * 32


def inputs(cid, lg, seed):
    n = 1 << lg
    base = msm.generate_points_dev(cid, 1 << min(lg, 16))
    pts = base.repeat(n // base.shape[0], 1).contiguous()
    g = torch.Generator(device="cuda").manual_seed(seed)
    s255 = torch.randint(-2**63, 2**63 - 1, (n, 4), dtype=torch.int64, device="cuda", generator=g)
    s64 = torch.randint(-2**63, 2**63 - 1, (n,), dtype=torch.int64, device="cuda", generator=g)
    return pts, s255, s64


def device_entry(rounds, lgs, curves):
    cases = [(c, lg, bits) for c in curves for lg in lgs for bits in (255, 64)]
    data, outs, times = {}, {}, {k: [] for k in cases}
    for c, lg, bits in cases:
        if (c, lg) not in data:
            data[(c, lg)] = inputs(CURVES[c], lg, lg)
            outs[(c, lg)] = torch.empty_like(data[(c, lg)][0])
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def call(c, lg, bits):
        pts, s255, s64 = data[(c, lg)]
        sc = s255 if bits == 255 else s64
        msm.scale_points_dev(CURVES[c], pts, sc, nbits=bits, out=outs[(c, lg)])

    for k in cases:                                                             # warm-up
        call(*k)
    torch.cuda.synchronize()
    for _ in range(rounds):
        for k in cases:
            ev0.record()
            call(*k)
            ev1.record()
            ev1.synchronize()
            times[k].append(ev0.elapsed_time(ev1))
    return [{"curve": c, "lg": lg, "bits": bits, "ms": stats(times[(c, lg, bits)])} for c, lg, bits in cases]


def host_entry(rounds):
    cid, lg = CURVES["bls12_381"], 20
    pts, s255, _ = inputs(cid, lg, 7)
    res = []
    page = (pts.cpu().numpy().view(np.uint64).copy(), s255.cpu().numpy().view(np.uint64).copy())
    pin_p = torch.empty(pts.shape, dtype=torch.int64, pin_memory=True)
    pin_s = torch.empty(s255.shape, dtype=torch.int64, pin_memory=True)
    pin_p.copy_(pts)
    pin_s.copy_(s255)
    pinned = (pin_p.numpy().view(np.uint64), pin_s.numpy().view(np.uint64))
    want = msm.scale_points_dev(cid, pts, s255).cpu().numpy().view(np.uint64)
    t = {"pageable": [], "pinned": []}
    same = True
    for name, (p, s) in (("pageable", page), ("pinned", pinned)):
        same &= bool(np.array_equal(msm.scale_points(cid, p, s), want))              # warm-up, checked
    for _ in range(rounds):
        for name, (p, s) in (("pageable", page), ("pinned", pinned)):
            t0 = time.perf_counter()
            msm.scale_points(cid, p, s)
            t[name].append((time.perf_counter() - t0) * 1e3)
    for name in t:
        res.append({"curve": "bls12_381", "lg": lg, "memory": name, "ms": stats(t[name]), "same_as_device": same})
    return res


def ladder_share():
    from torch.profiler import ProfilerActivity, profile
    cid, lg = CURVES["bls12_381"], 20
    pts, s255, _ = inputs(cid, lg, 9)
    out = torch.empty_like(pts)
    msm.scale_points_dev(cid, pts, s255, out=out)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        msm.scale_points_dev(cid, pts, s255, out=out)
        torch.cuda.synchronize()
    kern = {}
    for e in prof.events():
        if e.device_type.name == "CUDA":
            name = e.name.split("(")[0].split("<")[0].split()[-1]
            us = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
            kern[name] = kern.get(name, 0.0) + us / 1e3
    props = torch.cuda.get_device_properties(0)
    clk_khz = None
    try:
        import subprocess
        clk_khz = 1e3 * float(subprocess.check_output(
            ["nvidia-smi", "--query-gpu=clocks.max.sm", "--format=csv,noheader,nounits"], text=True).split()[0])
    except Exception:                                                           # noqa: BLE001
        pass
    mhz = clk_khz / 1e3 if clk_khz else 1980.0
    bound_ms = (1 << lg) * IMAD_PER_PRODUCT / (IMAD_RATE_PER_SM_CLK * props.multi_processor_count * mhz * 1e6) * 1e3
    ladder = sum(v for k, v in kern.items() if "scale_ladder" in k)
    return {"kernels_ms": kern, "ladder_ms": ladder, "bound_ms": bound_ms, "sm_clock_mhz": mhz,
            "sms": props.multi_processor_count, "share": bound_ms / ladder if ladder else None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--lgs", default="16,18,20,22")
    ap.add_argument("--curves", default=",".join(CURVES))
    ap.add_argument("--device-only", action="store_true")
    ap.add_argument("--out")
    a = ap.parse_args()
    gpu = card()
    print(f"# {gpu}", flush=True)
    dev = device_entry(a.rounds, [int(v) for v in a.lgs.split(",")], a.curves.split(","))
    for r in dev:
        m = r["ms"]
        rate = (1 << r["lg"]) / m["median"] / 1e3
        print(f"dev  {r['curve']:>13} 2^{r['lg']} {r['bits']:3d}-bit  {m['median']:10.3f} [{m['min']:.3f}, {m['max']:.3f}] ms"
              f"  {rate:8.3f} Mpoints/s", flush=True)
    if a.device_only:
        return
    host = host_entry(a.rounds)
    for r in host:
        m = r["ms"]
        print(f"host {r['curve']:>13} 2^{r['lg']} {r['memory']:>8}  {m['median']:10.3f} [{m['min']:.3f}, {m['max']:.3f}] ms"
              f"  same={r['same_as_device']}", flush=True)
    share = ladder_share()
    print(f"# kernels (profiler, BLS12-381 G1 2^20, 255-bit): " +
          " ".join(f"{k}={v:.3f}ms" for k, v in share["kernels_ms"].items()), flush=True)
    print(f"# IMAD.WIDE bound {share['bound_ms']:.1f} ms at {share['sm_clock_mhz']:.0f} MHz x {share['sms']} SMs;"
          f" ladder {share['ladder_ms']:.1f} ms; share {share['share']:.3f}" if share["share"] else "# no ladder kernel seen",
          flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump({"gpu": gpu, "device": dev, "host": host, "ladder": share}, f, indent=1)


if __name__ == "__main__":
    main()
