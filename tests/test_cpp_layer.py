"""The C++ surface (include/sppark_b200.hpp + include/compat/): layouts, that the headers compile,
and -- on a GPU -- that what the example program computes equals the oracle.  SURVEY.md section 8b,
"C++-level names to keep"."""
import ctypes as C
import importlib.util
import os
import random
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CPP = os.path.join(ROOT, "tests", "cpp")
OUT = os.path.join(CPP, "_build")
R_BLS = 0x73eda753299d7d483339d80809a1d80553bda402fffe5bfeffffffff00000001
GL_P = 2**64 - 2**32 + 1


def _builder():
    spec = importlib.util.spec_from_file_location("build_cpp", os.path.join(CPP, "build_cpp.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


@pytest.mark.parametrize("feature", ["BLS12_381", "PALLAS", "VESTA", "BN254", "BLS12_377", "GOLDILOCKS", "BABY_BEAR"])
def test_layouts_compile(feature):
    subprocess.check_call(["g++", "-std=c++17", "-fsyntax-only", f"-DFEATURE_{feature}", "-I" + os.path.join(ROOT, "include"),
                           os.path.join(CPP, "layout_check.cpp")])


@pytest.mark.parametrize("feature", ["GOLDILOCKS", "BABY_BEAR", "BLS12_381"])
def test_polynomial_headers_forward(feature):
    """<polynomial/prefix_op.cuh>, <polynomial/div_by_x_minus_z.cuh>, <polynomial/evaluate.cuh> and
    <ff/batch_inversion.hpp> resolve under include/compat to the same-named templates over the C ABI"""
    src = open(os.path.join(CPP, "poly_compat_check.cpp")).read()
    if feature != "GOLDILOCKS":
        src = src.replace("<ff/goldilocks.hpp>", "<ff/baby_bear.hpp>" if feature == "BABY_BEAR" else "<ff/bls12-381.hpp>")
    subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-x", "c++", f"-DFEATURE_{feature}",
                    "-I" + os.path.join(ROOT, "include", "compat"), "-"], input=src, text=True, check=True)


def test_unbuilt_curves_are_refused_at_compile_time():
    r = subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-DFEATURE_MERSENNE31", "-I" + os.path.join(ROOT, "include"),
                        os.path.join(CPP, "layout_check.cpp")], capture_output=True, text=True)
    assert r.returncode != 0 and "not instantiated" in r.stderr


def test_example_links_against_the_library(lib):
    exe, exe_ntt = _builder().build_example()
    assert os.path.exists(exe) and os.path.exists(exe_ntt)


class RE(C.Structure):
    _fields_ = [("code", C.c_int), ("message", C.c_void_p)]


def _limbs(x, n=4):
    return [(x >> (64 * i)) & 0xFFFFFFFFFFFFFFFF for i in range(n)]


def _scalars(n, seed):
    rnd = random.Random(seed)
    return np.array([_limbs(rnd.randrange(R_BLS)) for _ in range(n)], dtype=np.uint64).reshape(n, 4)


@pytest.mark.gpu
@pytest.mark.parametrize("mont", [0, 1])
def test_cpp_example_msm(oracle, tmp_path, mont):
    """mult_pippenger<bucket_t>(out, points, n, scalars, mont, sizeof(affine_t)) from C++; mont = 1
    is the template's default in the reference: scalars arrive as Montgomery residues."""
    exe, _ = _builder().build_example()
    n = 3000
    base = oracle.gen_points("bls12_381", 128)
    pts = np.zeros((n, 13), dtype=np.uint64)
    pts[:, :12] = base[np.arange(n) % 128]
    pts[5, 12] = 1
    sc = _scalars(n, 31 + mont)
    send = sc
    if mont:
        send = np.array([_limbs(oracle.ff_op("bls12_381_fr", "to_mont", sum(int(v) << (64 * j) for j, v in enumerate(row))))
                         for row in sc], dtype=np.uint64)
    pts.tofile(tmp_path / "p.bin")
    send.tofile(tmp_path / "s.bin")
    subprocess.check_call([exe, "msm", str(tmp_path / "p.bin"), str(tmp_path / "s.bin"), str(n), str(mont), str(tmp_path / "o.bin")])
    got = np.fromfile(tmp_path / "o.bin", dtype=np.uint64)
    ref = pts[:, :12].copy()
    ref[5] = 0
    want = oracle.msm("bls12_381", ref, sc, "pippenger", ncpus=8)
    assert np.array_equal(oracle.jac_to_affine("bls12_381", got), oracle.jac_to_affine("bls12_381", want))


@pytest.mark.gpu
def test_cpp_example_preloaded_points(oracle, tmp_path):
    """msm_t{points, npoints}.invoke(out, scalars): the SRS stays on the GPU between invocations."""
    exe, _ = _builder().build_example()
    n = 4000
    pts = np.zeros((n, 13), dtype=np.uint64)
    pts[:, :12] = oracle.gen_points("bls12_381", 128)[np.arange(n) % 128]
    sc = _scalars(n, 77)
    pts.tofile(tmp_path / "p.bin")
    sc.tofile(tmp_path / "s.bin")
    subprocess.check_call([exe, "ctx", str(tmp_path / "p.bin"), str(tmp_path / "s.bin"), str(n), "0", str(tmp_path / "o.bin")])
    got = np.fromfile(tmp_path / "o.bin", dtype=np.uint64).reshape(2, 18)
    flat = np.ascontiguousarray(pts[:, :12])
    for k, m in enumerate((n, n // 2)):
        want = oracle.msm("bls12_381", flat[:m], sc[:m], "pippenger", ncpus=8)
        assert np.array_equal(oracle.jac_to_affine("bls12_381", got[k]), oracle.jac_to_affine("bls12_381", want)), m


@pytest.mark.gpu
def test_cpp_example_ntt(oracle, tmp_path):
    _, exe = _builder().build_example()
    rng = np.random.default_rng(3)
    x = rng.integers(0, GL_P, size=1 << 12, dtype=np.uint64)
    x.tofile(tmp_path / "d.bin")
    subprocess.check_call([exe, "ntt", str(tmp_path / "d.bin"), "12", "0", "0", "1"])      # NN, forward, coset
    got = np.fromfile(tmp_path / "d.bin", dtype=np.uint64)
    assert np.array_equal(got, oracle.ntt_gl64(x, oracle.NN, False, True))
