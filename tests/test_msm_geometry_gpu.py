"""The device MSM at every window width, heavy-bucket split and slice schedule the host can choose
(csrc/msm/msm_core.cuh make_config / choose_wbits, msm.cuh msm_t, msm_host.cuh slice schedule).

Every result is compared, as an affine point, with a plain reference of the same sum: the C oracle
for G1 and BLS12-381 G2, oracle/g2py.py for BN254 and BLS12-377 G2.  Large inputs repeat m distinct
points, so the reference is the m-point MSM with the scalars summed per point mod r.

Every GPU case also checks that it ran the shape it claims to cover.  With SPPARK_B200_MSM_DEBUG=1
the MSM prints one line per slice: its size, the window width and count, the heavy threshold, and
how many heavy buckets and heavy chunks the sort registered.  Width, window count and threshold are
compared with make_config (compiled with g++ here), the heavy buckets and chunks with a NumPy
bucket count of the same scalars, slice by slice."""
import os
import re
import subprocess

import numpy as np
import pytest

from test_msm_sort import _digits

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# natural window width: (c, first point count that takes it); the range of c ends where the next
# row starts.  test_width_table_matches_make_config keeps it equal to the cost model.
WIDTHS = [(4, 1), (5, 133), (6, 300), (7, 820), (8, 1713), (9, 5497), (10, 9725), (11, 27907),
          (12, 50739), (13, 91330), (14, 365319), (16, 608865), (20, 10391294), (22, 90923820)]
LAST_N = (1 << 31) - 1                  # msm_t::begin rejects 2^31 points and more

CFG_SRC = r'''
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <algorithm>
#include "sppark_b200/csrc/msm/msm_core.cuh"
// "widths": every point count below 2^31 at which the chosen width changes, with the new width,
// found by bisection between the points of a geometric grid (step 0.2 %).  Otherwise: one line
// "wbits nwins heavy heavy_chunk" per point count given.
static uint32_t width(size_t n) { return msm::make_config(n).wbits; }
int main(int argc, char** argv)
{
    if (argc == 2 && !strcmp(argv[1], "widths")) {
        const size_t last = ((size_t)1 << 31) - 1;
        size_t prev = 1;
        uint32_t c = width(1);
        printf("%u 1\n", c);
        for (double x = 1.0; prev < last; x *= 1.002) {
            const size_t n = std::min<size_t>((size_t)x + 1, last);
            while (width(n) != c) {
                size_t lo = prev, hi = n;                   // width(lo) == c != width(hi)
                while (hi - lo > 1) {
                    const size_t mid = lo + (hi - lo) / 2;
                    (width(mid) == c ? lo : hi) = mid;
                }
                c = width(hi);
                prev = hi;
                printf("%u %zu\n", c, hi);
            }
            prev = n;
        }
        return 0;
    }
    for (int i = 1; i < argc; i++) {
        const msm::Config c = msm::make_config(strtoull(argv[i], nullptr, 10));
        printf("%u %u %u %u\n", c.wbits, c.nwins, c.heavy, c.heavy_chunk);
    }
    return 0;
}
'''


@pytest.fixture(scope="module")
def cfg_exe(tmp_path_factory):
    d = tmp_path_factory.mktemp("geometry")
    src, exe = d / "cfg.cpp", d / "cfg"
    src.write_text(CFG_SRC)
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-I", ROOT, "-I", "/usr/local/cuda/include", "-o", str(exe), str(src)])
    return str(exe)


def _make_config(exe, n):
    """make_config(n) under the current environment (the SPPARK_B200_MSM_* knobs a test has set)"""
    wbits, nwins, heavy, chunk = map(int, subprocess.check_output([exe, str(n)], text=True).split())
    return dict(wbits=wbits, nwins=nwins, heavy=heavy, heavy_chunk=chunk)


def test_width_table_matches_make_config(cfg_exe):
    """The GPU cases below take their sizes from WIDTHS: a change of the cost model must show up
    here, not leave them running at widths they no longer reach."""
    env = {k: v for k, v in os.environ.items() if not k.startswith("SPPARK_B200_MSM_")}
    rows = subprocess.check_output([cfg_exe, "widths"], text=True, env=env).split("\n")
    assert [tuple(int(v) for v in r.split()) for r in rows if r] == WIDTHS
    for (c, first), nxt in zip(WIDTHS, WIDTHS[1:] + [(None, LAST_N + 1)]):
        out = subprocess.check_output([cfg_exe, str(first), str(nxt[1] - 1)], text=True, env=env).split("\n")
        for line in out[:2]:
            wbits, nwins = map(int, line.split()[:2])
            assert (wbits, nwins) == (c, -(-256 // c))


def _natural_width(n):
    return [c for c, first in WIDTHS if first <= n][-1]


# ---- curves: distinct points, the reference sum, affine comparison -------------------------------
INF, NEG = 5, 7                 # distinct point INF is infinity, point NEG is -(point NEG - 1)
R_BLS = 0x73eda753299d7d483339d80809a1d80553bda402fffe5bfeffffffff00000001


def _int(row):
    return sum(int(v) << (64 * i) for i, v in enumerate(row))


def _limbs(x, n=4):
    return [(x >> (64 * i)) & 0xFFFFFFFFFFFFFFFF for i in range(n)]


def _neg_y(row, p, nl):
    """negate the Y half of a packed affine row (Fp or Fp2 coordinates, Montgomery form)"""
    out = row.copy()
    half = row.shape[0] // 2
    for k in range(half, row.shape[0], nl):
        v = _int(row[k:k + nl])
        out[k:k + nl] = _limbs((p - v) % p, nl)
    return out


class Curve:
    def __init__(self, oracle, name):
        from sppark_b200 import msm
        self.name, self.oracle = name, oracle
        self.g2py = None
        if name.endswith("_g2") and name != "bls12_381_g2":
            from oracle import g2py
            self.g2py = g2py.curve(name)
            self.cid, self.r = self.g2py.id, self.g2py.r
        else:
            self.cid = {"bls12_381": msm.BLS12_381_G1, "pallas": msm.PALLAS, "vesta": msm.VESTA,
                        "bn254": msm.BN254_G1, "bls12_377": msm.BLS12_377_G1, "bls12_381_g2": msm.BLS12_381_G2}[name]
            fr = {"bls12_381": "bls12_381_fr", "pallas": "vesta_fp", "vesta": "pallas_fp", "bn254": "bn254_fr",
                  "bls12_377": "bls12_377_fr", "bls12_381_g2": "bls12_381_fr"}[name]
            self.r = oracle.ff_consts(fr)["p"]
        self._bases = {}

    def base(self, m):
        """m distinct packed affine points, INF infinity and NEG = -(NEG - 1) when m is large enough"""
        if m not in self._bases:
            if self.g2py is not None:
                from oracle import g2py
                pts = g2py.multiples(self.g2py, m)
                if m > NEG:
                    pts[INF], pts[NEG] = None, self.g2py.neg(pts[NEG - 1])
                self._bases[m] = self.g2py.encode_affine(pts)
            else:
                fp = "bls12_381_fp" if self.name == "bls12_381_g2" else self.name + "_fp"
                p, nl = self.oracle.ff_consts(fp)["p"], self.oracle.FIELD_LIMBS[self.oracle.FIELDS[fp]]
                rows = self.oracle.g2_points(m) if self.name == "bls12_381_g2" else self.oracle.gen_points(self.name, m)
                if m > NEG:
                    rows[INF] = 0
                    rows[NEG] = _neg_y(rows[NEG - 1], p, nl)
                self._bases[m] = rows
        return self._bases[m]

    def reference(self, base, scalars):
        """sum_i scalars[i] * base[i], affine"""
        if self.g2py is not None:
            pts = self.g2py.decode_affine(base)
            return self.g2py.msm(pts, [_int(s) for s in scalars])
        if self.name == "bls12_381_g2":
            return self.affine(self.oracle.g2_msm(base, scalars))
        return self.affine(self.oracle.msm(self.name, base, scalars, "pippenger", ncpus=8))

    def affine(self, jac):
        if self.g2py is not None:
            return self.g2py.jacobian_to_affine(jac)
        if self.name == "bls12_381_g2":
            return tuple(self.oracle.g2_jac_to_affine(jac).tolist())
        return tuple(self.oracle.jac_to_affine(self.name, jac).tolist())


_CURVES = {}


def _curve(oracle, name):
    if name not in _CURVES:
        _CURVES[name] = Curve(oracle, name)
    return _CURVES[name]


# ---- scalars ----------------------------------------------------------------------------------
def _uniform(n, seed, r=None, bits=None):
    """uniform below 2^bits, or (top limb below r's) just below r"""
    rng = np.random.default_rng(seed)
    sc = rng.integers(0, 2**64, size=(n, 4), dtype=np.uint64)
    if bits is not None:
        sc[:, 3] >>= np.uint64(256 - bits)
    else:
        sc[:, 3] = rng.integers(0, r >> 192, size=n, dtype=np.uint64)
    return sc


def _special(c, r):
    """every digit +2^(c-1) (the highest bucket, the largest running-sum weight); every raw window
    2^(c-1) + 1 (a negative digit and a carry into every next window); 2^255 - 1; r - 1"""
    nwins, half = -(-256 // c), 1 << (c - 1)
    top = sum(half << (c * w) for w in range(nwins) if c * w + c - 1 < 255)
    neg = sum((half + 1) << (c * w) for w in range(nwins) if c * w + c <= 255)
    return [top, neg, (1 << 255) - 1, r - 1]


def _mixed(n, seed, c, r, m):
    """uniform scalars below r with the special values of width c in every 16th part of the rows,
    and equal scalars on the rows of the points NEG - 1 and NEG (they cancel)"""
    sc = _uniform(n, seed, r=r)
    stride = max(8, n // 16)
    for k, v in enumerate(_special(c, r)):
        sc[k::stride] = _limbs(v)
    rows = np.arange(NEG - 1, n - 1, m)
    sc[rows + 1] = sc[rows]
    return sc


def _top_plant(c, b):
    """a scalar with one non-zero digit: bucket b of the top window"""
    return _limbs((b + 1) << (c * (-(-256 // c) - 1)))


def _fold(sc, m, r):
    """per distinct point i: the sum of the scalars of the rows j = i mod m, mod r"""
    import bench
    pad = (-sc.shape[0]) % m
    if pad:
        sc = np.concatenate([sc, np.zeros((pad, 4), dtype=np.uint64)])
    return bench.fold_scalars(sc, m, r)


# ---- expected shape -----------------------------------------------------------------------------
LINE = re.compile(r"\[msm\] slice (\d+) n=(\d+) wbits=(\d+) nwins=(\d+) heavy_thr=(\d+) tasks_claimed=\d+ "
                  r"nheavy=(\d+) nchunks=(\d+)")


def _schedule(n, resident=False):
    """slice sizes of msm_host (the device-pointer entry runs one slice)"""
    if os.environ.get("SPPARK_B200_MSM_SLICES"):
        k = max(1, int(os.environ["SPPARK_B200_MSM_SLICES"]))
        each = ((n + k - 1) // k + 31) & ~31
        return [min(each, n - d) for d in range(0, n, each)]
    if resident and n >= 1 << 22:
        e = (n // 8 + 31) & ~31
        return [e, n - e]
    if n >= 1 << 22:
        e = (n // 16 + 31) & ~31
        return [e, 2 * e, 4 * e, n - 7 * e]
    return [n]


def _slot_counts(sc, c):
    """entries of every (window, bucket) slot of the signed c-bit recoding of these scalars
    (2^20-row groups on all cores; cache-sized pieces inside a group)"""
    from concurrent.futures import ThreadPoolExecutor
    nwins, nb = -(-256 // c), 1 << (c - 1)
    offs = (np.arange(nwins, dtype=np.int64) * nb)[:, None]

    def group(g):
        keys = []
        for a in range(g, min(g + (1 << 20), sc.shape[0]), 1 << 14):
            b, _ = _digits(np.ascontiguousarray(sc[a:a + (1 << 14)]).view(np.uint32), c)
            keys.append((b + offs)[b >= 0])
        return np.bincount(np.concatenate(keys), minlength=nwins * nb)

    counts = np.zeros(nwins * nb, dtype=np.int64)
    with ThreadPoolExecutor(min(8, os.cpu_count() or 1)) as pool:
        for part in pool.map(group, range(0, sc.shape[0], 1 << 20)):
            counts += part
    return counts


def _check_shape(err, exe, sc, c, sched):
    """the debug lines show width c and make_config's window count and threshold, one line per slice
    of `sched`, and per slice the heavy buckets / chunks the NumPy bucket counts predict.
    Returns the heavy-bucket count of every slice."""
    cfg = _make_config(exe, sc.shape[0])
    assert cfg["wbits"] == c, cfg
    lines = [tuple(map(int, t)) for t in LINE.findall(err)]
    assert len(lines) == len(sched), err[-2000:]
    first, heavy = 0, []
    for k, (line, part) in enumerate(zip(lines, sched)):
        assert line[:5] == (k, part, c, cfg["nwins"], cfg["heavy"]), (line, part, cfg)
        counts = _slot_counts(sc[first:first + part], c)
        h = counts[counts > cfg["heavy"]]
        want = (int(h.size), int(((h + cfg["heavy_chunk"] - 1) // cfg["heavy_chunk"]).sum()))
        assert line[5:] == want, (k, line, want, cfg)
        heavy.append(line[5])
        first += part
    return heavy


@pytest.fixture
def debug(monkeypatch, capfd):
    monkeypatch.setenv("SPPARK_B200_MSM_DEBUG", "1")
    for k in ("SPPARK_B200_MSM_WBITS", "SPPARK_B200_MSM_HEAVY", "SPPARK_B200_MSM_SLICES",
              "SPPARK_B200_MSM_SCHED", "SPPARK_B200_MSM_PAIR"):
        monkeypatch.delenv(k, raising=False)
    capfd.readouterr()
    return capfd


def _host_case(oracle, capfd, exe, curve, sc, c, m=512, want_heavy=False):
    """host-pointer MSM of sc against m distinct points repeated; shape and value checked"""
    from sppark_b200 import msm
    cv = _curve(oracle, curve)
    base = cv.base(m)
    n = sc.shape[0]
    capfd.readouterr()
    got = msm.msm(cv.cid, np.resize(base, (n, base.shape[1])), sc)
    heavy = _check_shape(capfd.readouterr().err, exe, sc, c, _schedule(n))
    if want_heavy:
        assert max(heavy) > 0, "no heavy bucket: the heavy kernels did not run"
    assert cv.affine(got) == cv.reference(base, _fold(sc, m, cv.r))
    return heavy


# ---- 2. every width the host picks, on every curve -------------------------------------------------
def _sweep_sizes():
    sizes = []
    for (c, first), nxt in zip(WIDTHS, WIDTHS[1:]):
        if first >= 10391294:
            break
        sizes += [(c, first), (c, nxt[1] - 1)]
    return sizes + [(20, 10391294)]


@pytest.mark.gpu
@pytest.mark.parametrize("c,n", _sweep_sizes())
def test_bls12_381_every_natural_width(oracle, debug, cfg_exe, c, n):
    """first and last point count of every width up to the first c = 20 count, special scalars mixed in"""
    assert _natural_width(n) == c
    _host_case(oracle, debug, cfg_exe, "bls12_381", _mixed(n, n, c, R_BLS, 512), c)


@pytest.mark.gpu
@pytest.mark.parametrize("lg", [17, 18, 19])
def test_bls12_381_prover_sizes(oracle, debug, cfg_exe, lg):
    """2^17..2^19 with scalars uniform below r: the top window goes through the heavy kernels"""
    n = 1 << lg
    c = _natural_width(n)
    _host_case(oracle, debug, cfg_exe, "bls12_381", _uniform(n, lg, r=R_BLS), c, want_heavy=True)


@pytest.mark.gpu
@pytest.mark.parametrize("curve", ["pallas", "vesta", "bn254", "bls12_377"])
@pytest.mark.parametrize("n", [300, 5497, 1 << 17, 1 << 19])
def test_g1_curves_widths(oracle, debug, cfg_exe, curve, n):
    """c = 6, 9, 13 and 14 on the other G1 curves"""
    c = _natural_width(n)
    cv = _curve(oracle, curve)
    _host_case(oracle, debug, cfg_exe, curve, _mixed(n, n + cv.cid, c, cv.r, 512), c, want_heavy=n >= 1 << 17)


@pytest.mark.gpu
@pytest.mark.parametrize("curve,m", [("bls12_381_g2", 256), ("bn254_g2", 32), ("bls12_377_g2", 32)])
@pytest.mark.parametrize("lg", [17, 19])
def test_g2_widths(oracle, debug, cfg_exe, curve, m, lg):
    """c = 13 and 14 on the three G2 groups (F::N = 24 for the BLS12 ones: 2 CTAs per SM, 16 four-lane
    groups per combine CTA)"""
    n = 1 << lg
    c = _natural_width(n)
    cv = _curve(oracle, curve)
    _host_case(oracle, debug, cfg_exe, curve, _mixed(n, lg + cv.cid, c, cv.r, m), c, m=m, want_heavy=True)


# ---- 3. heavy-bucket boundaries -------------------------------------------------------------------
# exact counts in top-window buckets of the 2^17 geometry (c = 13, threshold 256, chunk 2048) that
# scalars below 2^254 never reach (they stop at bucket 127)
PLANT_13 = {200: 256, 201: 257, 202: 2048, 203: 2049, 204: 3 * 2048}


@pytest.mark.gpu
@pytest.mark.parametrize("knob", [None, "0", "1", "2047", "2048"])
def test_heavy_boundaries(oracle, debug, monkeypatch, cfg_exe, knob):
    """counts at heavy, heavy + 1, heavy_chunk, heavy_chunk + 1 and 3 heavy_chunk; the threshold
    knob at 0 (every non-empty bucket heavy), 1, and just below and at a planted count"""
    if knob is not None:
        monkeypatch.setenv("SPPARK_B200_MSM_HEAVY", knob)
    n = 1 << 17
    cfg = _make_config(cfg_exe, n)
    assert (cfg["wbits"], cfg["heavy_chunk"]) == (13, 2048)
    assert cfg["heavy"] == (256 if knob is None else int(knob))
    sc = _uniform(n, 3, bits=254)
    rows = np.random.default_rng(4).permutation(n)
    k = 0
    for b, cnt in PLANT_13.items():
        sc[rows[k:k + cnt]] = _top_plant(13, b)
        k += cnt
    top = _slot_counts(sc, 13).reshape(20, 4096)[19]
    assert [int(top[b]) for b in PLANT_13] == list(PLANT_13.values())
    _host_case(oracle, debug, cfg_exe, "bls12_381", sc, 13, want_heavy=True)


# ---- 4. slices ---------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("nslices", [2, 3, 7])
@pytest.mark.parametrize("lg", [17, 19])
def test_slices(oracle, debug, monkeypatch, cfg_exe, nslices, lg):
    """host entry cut into slices that share the bucket file: bucket A heavy in even slices and light
    in odd ones, bucket B the other way round (merged through accumulate and through
    heavy_fold_kernel), bucket C only in the first slice (empty in every later one)"""
    monkeypatch.setenv("SPPARK_B200_MSM_SLICES", str(nslices))
    n = 1 << lg
    c = _natural_width(n)
    A, B, C = (210, 211, 212) if c == 13 else (4, 5, 6)     # top buckets no scalar below 2^254 reaches
    sc = _uniform(n, nslices + lg, bits=254)
    first = 0
    for s, part in enumerate(_schedule(n)):
        plant = [(A, 300 if s % 2 == 0 else 10), (B, 10 if s % 2 == 0 else 300)] + ([(C, 5)] if s == 0 else [])
        k = first
        for b, cnt in plant:
            sc[k:k + cnt] = _top_plant(c, b)
            k += cnt
        first += part
    heavy = _host_case(oracle, debug, cfg_exe, "bls12_381", sc, c, want_heavy=True)
    assert len(heavy) == nslices


# ---- 5. preloaded points, two-slice schedule from 2^22 invoked points ---------------------------------
@pytest.mark.gpu
def test_preloaded_points_2pow22(oracle, debug, cfg_exe):
    """MsmContext over 2^22 + 4096 points (packed and arkworks rows): invoked with all of them, with
    exactly 2^22 (the smallest count that takes the N/8 + rest schedule), with 2^22 - 1 (one slice),
    and with Montgomery-form scalars"""
    from sppark_b200 import msm
    m, n0 = 512, (1 << 22) + 4096
    cv = _curve(oracle, "bls12_381")
    base = cv.base(m)
    pts = np.resize(base, (n0, 12))
    ark = np.zeros((n0, 13), dtype=np.uint64)
    ark[:, :12] = pts
    ark[INF::m, :12] = 7                                # a flagged row's coordinates are ignored
    ark[INF::m, 12] = 1
    sc = _mixed(n0, 22, 16, R_BLS, m)
    # Montgomery-form scalars: 4099 distinct values, periodic
    t = _uniform(4099, 23, r=R_BLS)
    t_mont = np.array([_limbs(oracle.ff_op("bls12_381_fr", "to_mont", _int(row))) for row in t], dtype=np.uint64)
    period = np.arange(1 << 22) % 4099
    cases = [(n0, sc, None), (1 << 22, sc[:1 << 22], None), ((1 << 22) - 1, sc[:(1 << 22) - 1], None),
             (1 << 22, t[period], t_mont[period])]
    for layout in (pts, ark):
        ctx = msm.MsmContext(cv.cid, layout)
        try:
            for n, plain, mont in cases:
                debug.readouterr()
                got = ctx.invoke(np.ascontiguousarray(plain) if mont is None else mont, mont=mont is not None)
                sched = _schedule(n, resident=True)
                assert len(sched) == (2 if n >= 1 << 22 else 1)
                _check_shape(debug.readouterr().err, cfg_exe, plain, 16, sched)
                assert cv.affine(got) == cv.reference(base, _fold(plain, m, cv.r)), (layout.shape, n, mont is not None)
        finally:
            ctx.close()


# ---- 6. forced widths -------------------------------------------------------------------------------
def _need_device_bytes(need):
    import torch
    free, _ = torch.cuda.mem_get_info()
    if free < need:
        pytest.skip(f"needs {need / 2**30:.1f} GiB of device memory, {free / 2**30:.1f} GiB free")


@pytest.mark.gpu
@pytest.mark.parametrize("curve,c", [("bls12_381", c) for c in range(3, 25)] + [("pallas", c) for c in range(3, 21)]
                         + [("bls12_381_g2", c) for c in range(3, 21)])
def test_forced_width(oracle, debug, monkeypatch, cfg_exe, curve, c):
    """SPPARK_B200_MSM_WBITS at every value it accepts: zero-bit top windows (c = 3, 5, 15, 17), every
    combine radix (lg_nb mod 4) and every running-sum chunk lg_l = lg_nb - 12 from 0 to 11"""
    monkeypatch.setenv("SPPARK_B200_MSM_WBITS", str(c))
    cv = _curve(oracle, curve)
    bucket = {"bls12_381": 192, "pallas": 128, "bls12_381_g2": 384}[curve]    # bytes per XYZZ bucket
    _need_device_bytes((-(-256 // c) << (c - 1)) * bucket + (1 << 30))
    m = 256 if curve == "bls12_381_g2" else 512
    _host_case(oracle, debug, cfg_exe, curve, _mixed(4099, c, c, cv.r, m), c, m=m)


@pytest.mark.gpu
@pytest.mark.parametrize("c", [3, 13, 14])
def test_forced_width_pair_prereduction(oracle, debug, monkeypatch, cfg_exe, c):
    """SPPARK_B200_MSM_PAIR=1 (experimental): c = 3 loads the counts of all four buckets of a window
    as one uint4"""
    monkeypatch.setenv("SPPARK_B200_MSM_WBITS", str(c))
    monkeypatch.setenv("SPPARK_B200_MSM_PAIR", "1")
    _host_case(oracle, debug, cfg_exe, "bls12_381", _mixed(4099, 100 + c, c, R_BLS, 512), c)


# ---- 7. the largest sizes, device-resident ---------------------------------------------------------
def _dev_case(oracle, capfd, exe, sc, c, m=1024):
    import torch
    from sppark_b200 import msm
    n = sc.shape[0]
    nwins = -(-256 // c)
    # points, scalars, staging + sorted entries, buckets (msm_t::begin), and some slack
    _need_device_bytes(n * (96 + 32) + nwins * n * 12 + (nwins << (c - 1)) * 192 + (2 << 30))
    cv = _curve(oracle, "bls12_381")
    d_base = msm.generate_points_dev(cv.cid, m)
    try:
        dp = d_base.repeat(-(-n // m), 1)[:n]
        ds = torch.from_numpy(sc.view(np.int64)).cuda()
        capfd.readouterr()
        got = msm.msm_dev(cv.cid, dp, ds)
        err = capfd.readouterr().err
        base = d_base.cpu().numpy().view(np.uint64)
    finally:
        del d_base
        dp = ds = None
        torch.cuda.empty_cache()
    heavy = _check_shape(err, exe, sc, c, [n])
    assert cv.affine(got) == cv.reference(base, _fold(sc, m, cv.r))
    return heavy


@pytest.mark.gpu
def test_c20_c22_boundary(oracle, debug, cfg_exe):
    """the last c = 20 count and the first c = 22 count, on the same inputs plus one point"""
    n = WIDTHS[-1][1]
    sc = _uniform(n, 90, r=R_BLS)
    sc[1::7919] = _limbs((1 << 255) - 1)
    _dev_case(oracle, debug, cfg_exe, sc[:n - 1], 20)
    _dev_case(oracle, debug, cfg_exe, sc, 22)


@pytest.mark.gpu
@pytest.mark.parametrize("bits", [None, 254])
def test_2pow27(oracle, debug, cfg_exe, bits):
    """c = 22 at 2^27: heavy threshold and chunk both 16384.  Scalars below r put ~18k entries in
    each top bucket (two chunks); below 2^254, as bench.py draws them, ~32k (two or three chunks)"""
    n = 1 << 27
    cfg = _make_config(cfg_exe, n)
    assert (cfg["wbits"], cfg["heavy"], cfg["heavy_chunk"]) == (22, 16384, 16384)
    sc = _uniform(n, 27, r=R_BLS, bits=bits)
    heavy = _dev_case(oracle, debug, cfg_exe, sc, 22)
    assert heavy[0] > 0
