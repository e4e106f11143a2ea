"""MSM over small scalars on the CPU: the window chooser for a scalar bit bound (msm_core.cuh
make_config(n, nbits, scalar_bytes) / config_for_table, compiled with g++ here), the whole pipeline
with 4-, 8-, 16- and 32-byte scalars in the CPU single-stepper (tests/emu/msm_bits_emu.cpp) against the
oracle, and the argument checks of the three _bits entries of the C ABI."""
import ctypes as C
import os
import random
import subprocess

import numpy as np
import pytest

from test_emu import _build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
R_BLS = 0x73eda753299d7d483339d80809a1d80553bda402fffe5bfeffffffff00000001
NBITS = [1, 2, 8, 16, 31, 32, 33, 64, 65, 128, 200, 254, 255]

CFG_SRC = r'''
#include <cstdio>
#include <cstdlib>
#include <algorithm>
#include "sppark_b200/csrc/msm/msm_core.cuh"
// per (n, nbits) pair: make_config(n, nbits, 32), then make_config(n), then config_for_table(n, 13, 4, n, nbits, 8)
static void put(const msm::Config& c)
{   printf("%u %u %u %u %u %u %u %u ", c.wbits, c.nwins, msm::digit_count(c), c.heavy, c.heavy_chunk, c.copies,
           (unsigned)c.nbits, (unsigned)c.swords);   }
int main(int argc, char** argv)
{
    for (int i = 1; i + 1 < argc; i += 2) {
        const size_t n = strtoull(argv[i], nullptr, 10);
        const uint32_t nbits = atoi(argv[i + 1]);
        put(msm::make_config(n, nbits, 32));
        put(msm::make_config(n));
        put(msm::config_for_table(n, 13, 4, n, nbits, 8));
        printf("%u\n", msm::top_window_bits(msm::make_config(n, nbits, 32)));
    }
    return 0;
}
'''
FIELDS = ("wbits", "nwins", "digits", "heavy", "heavy_chunk", "copies", "nbits", "swords")


@pytest.fixture(scope="module")
def configs(tmp_path_factory):
    d = tmp_path_factory.mktemp("cfgbits")
    src, exe = d / "cfg.cpp", d / "cfg"
    src.write_text(CFG_SRC)
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-I", ROOT, "-I", "/usr/local/cuda/include", "-o", str(exe), str(src)])
    env = {k: v for k, v in os.environ.items() if not k.startswith("SPPARK_B200_MSM_")}
    args = [str(v) for lg in range(10, 29) for nb in NBITS for v in (1 << lg, nb)]
    rows = subprocess.check_output([str(exe), *args], text=True, env=env).split("\n")
    out = {}
    for (lg, nb), row in zip([(lg, nb) for lg in range(10, 29) for nb in NBITS], rows):
        v = list(map(int, row.split()))
        k = len(FIELDS)
        out[lg, nb] = (dict(zip(FIELDS, v[:k])), dict(zip(FIELDS, v[k:2 * k])), dict(zip(FIELDS, v[2 * k:3 * k])), v[-1])
    return out


def test_windows_cover_the_bound(configs):
    """W c >= nbits + 1 > (W - 1) c: the top digit never carries out, and no window is wasted"""
    for (lg, nb), (c, _, _, top) in configs.items():
        W, w = c["nwins"], c["wbits"]
        assert W == c["digits"] and W * w >= nb + 1 > (W - 1) * w, (lg, nb, c)
        assert 3 <= w <= 24 and 256 <= c["heavy"] <= 16384, (lg, nb, c)
        assert top == min(nb - (W - 1) * w, w - 1), (lg, nb, c, top)
        assert (c["nbits"], c["swords"], c["copies"]) == (nb, 8, 1)


def test_255_bits_is_todays_configuration(configs):
    for lg in range(10, 29):
        new, old, _, _ = configs[lg, 255]
        assert new == old, lg


def test_pinned_configurations(configs):
    """(wbits, nwins, heavy) chosen for 2^20 and 2^24 points with 1, 16 and 64-bit scalars"""
    want = {(20, 1): (4, 1, 256), (20, 16): (17, 1, 256), (20, 64): (13, 5, 256),
            (24, 1): (4, 1, 294), (24, 16): (17, 1, 294), (24, 64): (17, 4, 1177)}
    for key, v in want.items():
        c = configs[key][0]
        assert (c["wbits"], c["nwins"], c["heavy"]) == v, (key, c)


def test_table_keeps_width_and_sets(configs):
    """a c = 13 table with 4 copies (D = 20 digits, V = 5 sets): D_b digits read from ceil(D_b / V)
    copies; with D_b <= V only copy 0, as the plain geometry of width 13"""
    for nb in NBITS:
        t = configs[20, nb][2]
        Db = (nb + 13) // 13
        assert (t["wbits"], t["digits"], t["swords"]) == (13, Db, 2)
        if Db <= 5:
            assert (t["nwins"], t["copies"]) == (Db, 1), (nb, t)
        else:
            assert (t["nwins"], t["copies"]) == (5, -(-Db // 5)), (nb, t)
    assert configs[20, 255][2]["copies"] == 4


# ---- the whole pipeline on the CPU ------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu():
    l = _build("msm_bits_emu")
    l.emu_msm_bls12_381_bits.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_uint, C.c_uint,
                                         C.c_uint, C.c_uint, C.c_uint]
    return l


def _pack(vals, sbytes):
    """little-endian scalars of sbytes bytes each, as the entries take them"""
    return np.frombuffer(b"".join(v.to_bytes(sbytes, "little") for v in vals), dtype=np.uint8).copy()


def _rows(vals):
    return np.array([[(v >> (64 * i)) & (2**64 - 1) for i in range(4)] for v in vals], dtype=np.uint64).reshape(-1, 4)


def _check(oracle, emu, pts, vals, sbytes, nbits, wbits, heavy=0, nslices=1):
    """the emulated MSM of vals (random bits above nbits included) against the oracle on vals mod 2^nbits"""
    sc = _pack(vals, sbytes)
    out = np.zeros(18, dtype=np.uint64)
    emu.emu_msm_bls12_381_bits(out.ctypes.data, pts.ctypes.data, pts.shape[0], sc.ctypes.data, sbytes, nbits,
                               wbits, heavy, nslices)
    want = oracle.msm("bls12_381", pts, _rows([v % (1 << nbits) for v in vals]), "pippenger", ncpus=4)
    return np.array_equal(oracle.jac_to_affine("bls12_381", out), oracle.jac_to_affine("bls12_381", want))


CASES = [  # (scalar_bytes, nbits, wbits): 0 = the chooser's width; widths that divide nbits leave a carry-only top window
    (4, 1, 0), (4, 1, 3), (4, 2, 0), (4, 8, 4), (4, 8, 8), (4, 16, 8), (4, 16, 16), (4, 31, 5), (4, 32, 8),
    (4, 32, 16), (8, 33, 11), (8, 63, 9), (8, 64, 16), (8, 64, 4), (16, 65, 13), (16, 100, 10), (16, 128, 16),
    (16, 128, 7), (32, 129, 3), (32, 200, 12), (32, 254, 0), (32, 255, 5), (32, 255, 11), (32, 64, 8), (8, 1, 12)]


@pytest.mark.parametrize("sbytes,nbits,wbits", CASES)
def test_pipeline_small_scalars(oracle, emu, sbytes, nbits, wbits):
    rnd = random.Random(sbytes * 1000 + nbits * 31 + wbits)
    n = 257
    pts = oracle.gen_points("bls12_381", 32)[np.arange(n) % 32].copy()
    pts[3] = 0
    vals = [rnd.randrange(1 << (8 * sbytes)) for _ in range(n)]      # random bits above nbits
    assert _check(oracle, emu, pts, vals, sbytes, nbits, wbits)


@pytest.mark.parametrize("sbytes,nbits,wbits", [(4, 16, 8), (4, 16, 5), (8, 64, 16), (8, 33, 11), (16, 128, 8),
                                                (4, 1, 4), (32, 255, 5)])
def test_pipeline_extreme_scalars(oracle, emu, sbytes, nbits, wbits):
    """every scalar 2^nbits - 1 (a carry through every window) or 2^(nbits - 1) (one top bucket), with
    random bits above; the buckets are heavy (threshold 4) and the points come in three slices"""
    rnd = random.Random(nbits + wbits)
    n = 150
    pts = oracle.gen_points("bls12_381", 8)[np.arange(n) % 8].copy()
    top = ((1 << (8 * sbytes)) - 1) ^ ((1 << nbits) - 1)
    for v in ((1 << nbits) - 1, 1 << (nbits - 1)):
        vals = [v | (rnd.getrandbits(8 * sbytes) & top) for _ in range(n)]
        assert _check(oracle, emu, pts, vals, sbytes, nbits, wbits, heavy=4, nslices=3), hex(v)


# ---- C ABI: argument checks before any device work --------------------------------------------------
BAD = [(3, 8), (12, 8), (64, 8), (0, 1), (4, 0), (8, 0), (4, 33), (8, 65), (16, 129), (32, 256), (32, 0)]
OK = [(4, 1), (4, 32), (8, 64), (16, 128), (32, 255)]
INVALID, NO_DEVICE = -1, -100


def _drop(lib, err):
    if err.message:
        lib.drop_error_message(err.message)
    return err.code


def _host_call(lib, sbytes, nbits, out, n=4):
    pts = np.zeros((n, 12), dtype=np.uint64)
    sc = np.zeros(n * 32, dtype=np.uint8)
    return _drop(lib, lib.sppark_b200_msm_bits(0, out.ctypes.data, pts.ctypes.data, n, sc.ctypes.data, 0, sbytes, nbits))


def _dev_call(lib, sbytes, nbits, out, ptr=0x10000):
    return _drop(lib, lib.sppark_b200_msm_dev_bits(0, out.ctypes.data, ptr, 4, ptr, sbytes, nbits, None))


@pytest.mark.parametrize("sbytes,nbits", BAD)
def test_bad_scalar_format_refused(lib, sbytes, nbits):
    """every entry refuses with -cudaErrorInvalidValue and writes infinity, without touching the device
    (the device pointers here are never dereferenced)"""
    for call in (_host_call, _dev_call):
        out = np.ones(18, dtype=np.uint64)
        assert call(lib, sbytes, nbits, out) == INVALID, call.__name__
        assert not out.any()
    out = np.ones(18, dtype=np.uint64)
    sc = np.zeros(128, dtype=np.uint8)
    assert _drop(lib, lib.sppark_b200_msm_ctx_invoke_bits(None, out.ctypes.data, sc.ctypes.data, 4, sbytes, nbits)) == INVALID


def test_misaligned_device_scalars_refused(lib):
    for sbytes in (8, 16, 32):
        out = np.ones(18, dtype=np.uint64)
        assert _dev_call(lib, sbytes, 8, out, ptr=0x10004) == INVALID
        assert not out.any()


@pytest.mark.parametrize("sbytes,nbits", OK)
def test_valid_format_needs_a_device(lib, sbytes, nbits):
    import torch
    if torch.cuda.is_available():
        pytest.skip("needs a CPU-only host")
    out = np.ones(18, dtype=np.uint64)
    assert _host_call(lib, sbytes, nbits, out) == NO_DEVICE
    assert _dev_call(lib, sbytes, nbits, out) == NO_DEVICE


def test_python_scalar_formats():
    """the width follows the array; mont=True goes with (n, 4) scalars and no bound only"""
    from sppark_b200 import msm
    u64, u32 = np.uint64, np.uint32
    assert msm._scalar_bytes(np.zeros((3, 4), u64), u64, u32) == 32
    assert msm._scalar_bytes(np.zeros((3, 2), u64), u64, u32) == 16
    assert msm._scalar_bytes(np.zeros(3, u64), u64, u32) == 8
    assert msm._scalar_bytes(np.zeros(3, u32), u64, u32) == 4
    assert msm._scalar_bytes(np.zeros((3, 3), u64), u64, u32) is None
    assert msm._scalar_format(32, True, None) is None
    assert msm._scalar_format(8, False, None) == (8, 64)
    assert msm._scalar_format(32, False, 16) == (32, 16)
    assert msm._scalar_format(4, False, None) == (4, 32)
    with pytest.raises(ValueError):
        msm._scalar_format(8, True, None)
    with pytest.raises(ValueError):
        msm._scalar_format(32, True, 64)
    with pytest.raises(ValueError):
        msm._scalar_format(4, False, 33)
    with pytest.raises(ValueError):
        msm._scalar_format(32, False, 0)
    pts = np.zeros((3, 12), u64)
    with pytest.raises(ValueError):
        msm.msm(msm.BLS12_381_G1, pts, np.zeros(3, u64), mont=True)
    with pytest.raises(ValueError):
        msm.msm(msm.BLS12_381_G1, pts, np.zeros(2, u32))
