"""In-tree build of libsppark_b200.so (nvcc, sm_90a only).

`python -m sppark_b200.build` or `__graft_entry__.build()`.  The .so and the objects under
build/ are build products (git-ignored).
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.environ.get("SPPARK_B200_LIB") or os.path.join(HERE, "libsppark_b200.so")   # override: experiments only

SOURCES = ["api.cu", "util/gpu.cu", "ntt/ntt.cu", "ntt/ntt_warp.cu", "poly/poly.cu", "msm/msm.cu", "msm/msm_bls12_381.cu", "msm/msm_bls12_381_g2.cu",
           "msm/msm_pasta.cu", "msm/msm_bn254_bls12_377.cu", "msm/msm_bn254_g2.cu", "msm/msm_bls12_377_g2.cu"]
# the Karatsuba product of the hot loop (ff/mont.cuh, SPPARK_B200_KARATSUBA) stays compiled out: on
# H100 it made the BLS12-381 G1 accumulate kernel slower than the fused ladder (DESIGN.md section
# 7.2).  Squaring and a*b - c*d use the fused ladder's own forms
NVCC_FLAGS = ["-std=c++17", "-O3", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo",
              "-Xcompiler", "-fPIC", "--threads", "4"]


def _sources():
    paths = [os.path.join(CSRC, s) for s in SOURCES]
    missing = [p for p in paths if not os.path.exists(p)]
    if missing:
        raise FileNotFoundError("missing sources: " + ", ".join(missing))
    return paths


def _newest_input():
    newest = 0.0
    for root, _, files in os.walk(CSRC):
        for f in files:
            newest = max(newest, os.path.getmtime(os.path.join(root, f)))
    inc = os.path.join(os.path.dirname(HERE), "include", "sppark_b200.h")
    return max(newest, os.path.getmtime(inc))


def _up_to_date(obj, flags):
    """Object newer than every file of its nvcc -MD dependency list, built with the same flags."""
    dep = obj[:-2] + ".d"
    try:
        if open(obj + ".flags").read() != " ".join(flags):
            return False
        t = os.path.getmtime(obj)
        words = open(dep).read().replace("\\\n", " ").split()
        return all(os.path.getmtime(w) <= t for w in words[1:] if not w.endswith(":"))
    except OSError:
        return False


def build(force=False, verbose=False):
    if not force and os.path.exists(LIB) and os.path.getmtime(LIB) >= _newest_input():
        return LIB
    objs = []
    procs = []
    extra = os.environ.get("SPPARK_B200_NVCC_EXTRA", "").split()
    objdir = os.path.join(HERE, "build" + ("_" + os.path.basename(LIB) if extra else ""))
    os.makedirs(objdir, exist_ok=True)
    for src in _sources():
        obj = os.path.join(objdir, os.path.basename(src).replace(".cu", ".o"))
        objs.append(obj)
        if not force and not verbose and _up_to_date(obj, [*NVCC_FLAGS, *extra]):
            continue
        cmd = ["nvcc", *NVCC_FLAGS, *extra, "-MD", "-c", "-o", obj, src]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        with open(obj + ".flags", "w") as f:
            f.write(" ".join([*NVCC_FLAGS, *extra]))
        procs.append((subprocess.Popen(cmd), cmd))
    for p, cmd in procs:
        if p.wait() != 0:
            raise RuntimeError("nvcc failed: " + " ".join(cmd))
    # --no-undefined: a symbol that is declared but that no object defines fails the link, not the
    # library's load
    subprocess.check_call(["nvcc", "-shared", "-o", LIB, *objs, "-gencode", "arch=compute_90a,code=sm_90a",
                           "-Xlinker", "--no-undefined"])
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
