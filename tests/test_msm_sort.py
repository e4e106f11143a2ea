"""The MSM's bucket sort (msm_core.cuh "sort", msm.cuh sort_slice) against a plain NumPy sort.

Exact: counts and (window-local) offsets of every (window, bucket) slot.  As sets: the entries of
each bucket (point index | sign << 31) and the list of heavy buckets.  The CPU single-stepper runs
the kernel bodies with a small bin capacity, so that bins also go down the overflow path; the GPU
tests run the device sort through a test-only entry at 2^20 and 2^22 points."""
import ctypes as C

import numpy as np
import pytest

from test_emu import _build

R_BLS = 0x73eda753299d7d483339d80809a1d80553bda402fffe5bfeffffffff00000001


def _digits(sc32, wbits):
    """(nwins, n) bucket indices (-1 for a zero digit) and signs of the signed c-bit recoding
    (msm_core.cuh Digits: bit 255 ignored, digits in (-2^(c-1), 2^(c-1)])."""
    n = sc32.shape[0]
    words = np.zeros((n, 10), dtype=np.uint64)
    words[:, :8] = sc32
    words[:, 7] &= np.uint64(0x7fffffff)
    nwins = (256 + wbits - 1) // wbits
    carry = np.zeros(n, dtype=np.uint64)
    half, full = np.uint64(1 << (wbits - 1)), np.uint64(1 << wbits)
    buckets, signs = np.empty((nwins, n), dtype=np.int64), np.empty((nwins, n), dtype=np.uint64)
    for w in range(nwins):
        off = w * wbits
        i, sh = off >> 5, off & 31
        both = words[:, i] | (words[:, i + 1] << np.uint64(32))
        raw = ((both >> np.uint64(sh)) & (full - np.uint64(1))) + carry
        neg = raw > half
        raw = np.where(neg, full - raw, raw)
        carry = neg.astype(np.uint64)
        buckets[w] = raw.astype(np.int64) - 1
        signs[w] = neg.astype(np.uint64)
    return buckets, signs


def _reference(sc32, wbits, heavy):
    n = sc32.shape[0]
    buckets, signs = _digits(sc32, wbits)
    nwins, nb = buckets.shape[0], 1 << (wbits - 1)
    counts = np.zeros((nwins, nb), dtype=np.uint32)
    offsets = np.zeros((nwins, nb), dtype=np.uint32)
    keys = []
    idx = np.arange(n, dtype=np.uint64)
    for w in range(nwins):
        nz = buckets[w] >= 0
        counts[w] = np.bincount(buckets[w][nz], minlength=nb)
        offsets[w] = np.cumsum(counts[w], dtype=np.uint32) - counts[w]
        slot = np.uint64(w * nb) + buckets[w][nz].astype(np.uint64)
        keys.append((slot << np.uint64(32)) | idx[nz] | (signs[w][nz] << np.uint64(31)))
    heavy_set = set(np.flatnonzero(counts.reshape(-1) > heavy).tolist())
    return counts.reshape(-1), offsets.reshape(-1), np.sort(np.concatenate(keys)), heavy_set


def _keys_from(counts, offsets, sorted_, nwins, nb, n):
    """(slot << 32 | entry) for every entry the sort placed, read back through counts / offsets."""
    keys = []
    c2, o2 = counts.reshape(nwins, nb).astype(np.int64), offsets.reshape(nwins, nb).astype(np.int64)
    for w in range(nwins):
        cw = c2[w]
        nzb = np.flatnonzero(cw)
        if nzb.size == 0:
            continue
        reps = cw[nzb]
        starts = np.repeat(o2[w][nzb], reps)
        within = np.arange(reps.sum()) - np.repeat(np.cumsum(reps) - reps, reps)
        pos = w * n + starts + within
        slot = np.repeat((w * nb + nzb).astype(np.uint64), reps)
        keys.append((slot << np.uint64(32)) | sorted_[pos].astype(np.uint64))
    return np.sort(np.concatenate(keys)) if keys else np.zeros(0, dtype=np.uint64)


def _check(got, sc32, wbits):
    counts, offsets, sorted_, heavy_slots, info = got
    n = sc32.shape[0]
    nwins, nb = (256 + wbits - 1) // wbits, 1 << (wbits - 1)
    assert info[0] == nwins
    want_c, want_o, want_keys, want_heavy = _reference(sc32, wbits, int(info[1]))
    assert np.array_equal(counts, want_c)
    assert np.array_equal(offsets, want_o)
    assert np.array_equal(_keys_from(counts, offsets, sorted_, nwins, nb, n), want_keys)
    assert set(heavy_slots[: info[2]].tolist()) == want_heavy
    assert info[2] == len(want_heavy)


@pytest.fixture(scope="module")
def emu():
    l = _build("msm_sort_emu")
    l.emu_msm_sort.argtypes = [C.c_size_t, C.c_uint, C.c_uint, C.c_uint] + [C.c_void_p] * 6
    return l


def _emu_sort(emu, sc32, wbits, heavy, cap):
    n = sc32.shape[0]
    nwins, nb = (256 + wbits - 1) // wbits, 1 << (wbits - 1)
    counts, offsets = np.zeros(nwins * nb, dtype=np.uint32), np.zeros(nwins * nb, dtype=np.uint32)
    sorted_, heavy_slots = np.zeros(nwins * n, dtype=np.uint32), np.zeros(nwins * n + 1, dtype=np.uint32)
    info = np.zeros(5, dtype=np.uint32)
    sc32 = np.ascontiguousarray(sc32, dtype=np.uint32)
    emu.emu_msm_sort(n, wbits, heavy, cap, sc32.ctypes.data, counts.ctypes.data, offsets.ctypes.data,
                     sorted_.ctypes.data, heavy_slots.ctypes.data, info.ctypes.data)
    return counts, offsets, sorted_, heavy_slots, info


def _scalars(kind, n, seed):
    rng = np.random.default_rng(seed)
    if kind == "uniform":
        sc = rng.integers(0, 2**32, size=(n, 8), dtype=np.uint64).astype(np.uint32)
        sc[:, 7] >>= 2                                          # below 2^254, as bench.py draws them
    elif kind == "top_bit":                                     # bit 255 set everywhere: ignored
        sc = rng.integers(0, 2**32, size=(n, 8), dtype=np.uint64).astype(np.uint32)
        sc[:, 7] |= 0x80000000
    elif kind == "zero":
        sc = np.zeros((n, 8), dtype=np.uint32)
    elif kind == "equal":
        sc = np.tile(np.array([(R_BLS - 1) >> (32 * k) & 0xffffffff for k in range(8)], dtype=np.uint32), (n, 1))
    elif kind == "two_valued":
        a = np.array([(R_BLS - 5) >> (32 * k) & 0xffffffff for k in range(8)], dtype=np.uint32)
        b = np.array([3, 0, 0, 0, 0, 0, 0, 0], dtype=np.uint32)
        sc = np.where(rng.integers(0, 2, size=(n, 1)) == 1, a, b).astype(np.uint32)
    else:                                                       # all ones: every digit negative
        sc = np.full((n, 8), 0xffffffff, dtype=np.uint32)
    return np.ascontiguousarray(sc)


@pytest.mark.parametrize("wbits", list(range(3, 25)))
@pytest.mark.parametrize("n", [1, 2, 33, 300, 5000])
def test_emulated_sort_uniform(emu, wbits, n):
    if (wbits >= 20 and n > 300) or (wbits >= 23 and n > 33):
        pytest.skip("the 2^(c-1) slots per window, not the points, set the cost here: covered at smaller n")
    sc = _scalars("uniform", n, 1000 * wbits + n)
    _check(_emu_sort(emu, sc, wbits, 0, 64), sc, wbits)


@pytest.mark.parametrize("kind", ["zero", "equal", "two_valued", "top_bit", "ones"])
@pytest.mark.parametrize("wbits", [3, 5, 8, 13, 16])
def test_emulated_sort_adversarial(emu, kind, wbits):
    """a bucket holding every entry of its window (far over the bin capacity), empty windows,
    bit 255 set, every digit negative"""
    sc = _scalars(kind, 3000, wbits)
    _check(_emu_sort(emu, sc, wbits, 50, 64), sc, wbits)


@pytest.mark.parametrize("cap", [1, 16, 1 << 20])
def test_emulated_sort_bin_capacity(emu, cap):
    """every bin over capacity (cap 1), some (16), none: the same lists"""
    sc = _scalars("uniform", 4000, cap)
    got = _emu_sort(emu, sc, 9, 30, cap)
    _check(got, sc, 9)
    if cap == 1:
        assert got[4][4] > 0
    if cap == 1 << 20:
        assert got[4][4] == 0


def test_emulated_sort_slices(emu):
    """an MSM cut into slices sorts each slice on its own, in the geometry of the whole MSM (the
    buckets are merged later, by accumulation: test_emu.py::test_msm_sliced_bucket_merging)"""
    sc = _scalars("uniform", 5000, 3)
    for a, b in [(0, 700), (700, 2000), (2000, 5000)]:
        part = np.ascontiguousarray(sc[a:b])
        _check(_emu_sort(emu, part, 10, 40, 64), part, 10)


def test_emulated_sort_top_window_bins(emu):
    """the narrow top window gets its own bin width: at c = 20 its buckets are < 2^15"""
    sc = _scalars("uniform", 5000, 7)
    counts, offsets, *_ = got = _emu_sort(emu, sc, 20, 0, 64)
    _check(got, sc, 20)
    top = counts.reshape(13, 1 << 19)[12]
    assert not top[1 << 15:].any()
    assert (offsets.reshape(13, 1 << 19)[12][1 << 15:] == 5000).all()


def _gpu_sort(sc32, wbits, cap=0):
    from sppark_b200 import _lib
    n = sc32.shape[0]
    nwins, nb = (256 + wbits - 1) // wbits, 1 << (wbits - 1)
    counts, offsets = np.zeros(nwins * nb, dtype=np.uint32), np.zeros(nwins * nb, dtype=np.uint32)
    sorted_, heavy_slots = np.zeros(nwins * n, dtype=np.uint32), np.zeros(nwins * n + 1, dtype=np.uint32)
    info = np.zeros(5, dtype=np.uint32)
    sc32 = np.ascontiguousarray(sc32, dtype=np.uint32)
    _lib.check(_lib.lib().sppark_b200_selftest_msm_sort(n, wbits, cap, sc32.ctypes.data, counts.ctypes.data,
                                                        offsets.ctypes.data, sorted_.ctypes.data,
                                                        heavy_slots.ctypes.data, info.ctypes.data))
    return counts, offsets, sorted_, heavy_slots, info


@pytest.mark.gpu
@pytest.mark.parametrize("lg", [20, 22])
@pytest.mark.parametrize("kind", ["uniform", "equal", "two_valued", "skewed"])
def test_device_sort(kind, lg):
    """uniform, all equal, two values, and skewed: half the points share one scalar, the other
    half draw from 64 values"""
    n = 1 << lg
    wbits = 16 if lg == 20 else 18
    if kind == "skewed":
        sc = _scalars("uniform", n, lg)
        sc[: n // 2] = sc[0]
        rng = np.random.default_rng(lg)
        sc[n // 2:] = sc[n // 2 + rng.integers(0, 64, size=n - n // 2)]
    else:
        sc = _scalars(kind, n, lg)
    got = _gpu_sort(sc, wbits)
    _check(got, sc, wbits)
    if kind in ("equal", "two_valued"):
        assert got[4][4] > 0


@pytest.mark.gpu
@pytest.mark.parametrize("wbits,cap", [(13, 256), (20, 1024), (8, 1 << 14)])
def test_device_sort_overflow_and_widths(wbits, cap):
    """a small bin capacity sends uniform bins down the overflow path; other window widths"""
    sc = _scalars("uniform", 1 << 18, wbits)
    got = _gpu_sort(sc, wbits, cap)
    _check(got, sc, wbits)
    assert got[4][4] > 0
