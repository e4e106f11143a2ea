"""Builds the C++-layer test programs (tests/test_cpp_layer.py, __graft_entry__.build()):
  _build/dropin_example        tests/cpp/dropin_example.cpp against include/sppark_b200.hpp
"""
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, "_build")
LINK = ["-L" + os.path.join(ROOT, "sppark_b200"), "-lsppark_b200", "-Wl,-rpath," + os.path.join(ROOT, "sppark_b200"),
        "-Wl,-rpath,$ORIGIN/../../../sppark_b200"]

def build_example():
    os.makedirs(OUT, exist_ok=True)
    exe = os.path.join(OUT, "dropin_example")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-DFEATURE_BLS12_381", "-I" + os.path.join(ROOT, "include"),
                           "-o", exe, os.path.join(HERE, "dropin_example.cpp"), *LINK])
    exe_ntt = os.path.join(OUT, "dropin_example_gl64")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-DFEATURE_GOLDILOCKS", "-DNTT_ONLY", "-I" + os.path.join(ROOT, "include"),
                           "-o", exe_ntt, os.path.join(HERE, "dropin_example.cpp"), *LINK])
    return exe, exe_ntt


if __name__ == "__main__":
    print(build_example())
