"""GPU: Goldilocks transforms on non-canonical input words, and coset transforms / LDE at the
sizes where the coset and twiddle tables change level.

A Goldilocks input word may be any uint64 and stands for its value mod p; every output word must
be canonical.  Each check compares bit-exactly with the CPU oracle on x % p, across both pass
kernels (warp-autonomous below 2^20, block-tile at 2^1..2^3 and from 2^20 on, each also forced to
the other side of that line), the host, device and batched entries, LDE, the slab-sharded passes
and the polynomial helpers.  The coset tables hold g^i, g^(i << 12) and g^(i << 24): 2^25-point
cosets are the first to use the third one."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

GL_P = 2**64 - 2**32 + 1
BB_P = 0x78000001
NN, NR, RN, RR = 0, 1, 2, 3
CORNERS = np.array([0, 1, GL_P - 1, GL_P, GL_P + 1, 2**64 - 1], dtype=np.uint64)


def loose_words(shape, seed):
    """Words that reach the carry corners of add/sub.  Along the last axis, the first half mixes
    words in [p, 2^64), in [0, 2^32), the corners and canonical words; the second half lies in
    [p, 2^64).  The first butterfly of a natural-order transform pairs i with i + n/2, so it meets
    two large words (their sum can wrap 2^64 twice) or a small and a large one (their difference
    can borrow twice); words 0, n/2 - 1, n/2 and n - 1 make both certain ([2^64 - 1, 2^64 - 1]
    when n = 2)."""
    rng = np.random.default_rng(seed)
    high = np.uint64(GL_P) + rng.integers(0, 2**32 - 1, size=shape, dtype=np.uint64)
    low = rng.integers(0, 2**32, size=shape, dtype=np.uint64)
    canon = rng.integers(0, GL_P, size=shape, dtype=np.uint64)
    corner = CORNERS[rng.integers(0, len(CORNERS), size=shape)]
    x = np.choose(rng.integers(0, 4, size=shape), [high, low, canon, corner])
    h = x.shape[-1] // 2
    x[..., h:] = high[..., h:]
    x[..., h - 1] = x[..., -1] = np.uint64(2**64 - 1)
    if h > 1:
        x[..., 0], x[..., h] = np.uint64(0), np.uint64(2**64 - 1)
    return x


def _reduce(x):
    return np.where(x >= np.uint64(GL_P), x - np.uint64(GL_P), x)


def _rand(field, n, seed):
    rng = np.random.default_rng(seed)
    if field == "gl64":
        return rng.integers(0, GL_P, size=n, dtype=np.uint64)
    return rng.integers(0, BB_P, size=n, dtype=np.uint32)


BREV8 = np.array([int(f"{b:08b}"[::-1], 2) for b in range(256)], dtype=np.uint32)


def _brev(lg):
    """the lg-bit bit-reversal permutation (32-bit reversal by bytes, shifted down)"""
    i = np.arange(1 << lg, dtype=np.uint32)
    r = (BREV8[i & 255] << 24) | (BREV8[(i >> 8) & 255] << 16) | (BREV8[(i >> 16) & 255] << 8) | BREV8[i >> 24]
    return (r >> np.uint32(32 - lg)).astype(np.int64)


def _cases(oracle, x, inverse, coset):
    """{order: (input, expected output)} for the four orders from one oracle transform of x % p
    (two for RR cosets, whose exponents are bit-reversed on natural-order data).  NR is the NN
    result bit-reversed; RN and its NN twin agree when RN is handed the bit-reversed input."""
    lg = x.size.bit_length() - 1
    xr = _reduce(x)
    r = _brev(lg)
    want = oracle.ntt_gl64(xr, NN, inverse, coset, nthreads=16)
    rr = oracle.ntt_gl64(xr, RR, inverse, True, nthreads=16) if coset else want
    return {NN: (x, want), NR: (x, want[r]), RN: (np.ascontiguousarray(x[r]), want), RR: (x, rr)}


def _check(got, want, *ctx):
    assert (got < np.uint64(GL_P)).all(), ("non-canonical output",) + ctx
    assert np.array_equal(got, want), ctx


def _host_entries(oracle, lg, seed):
    """compute_ntt and sppark_b200_ntt (field 0), every order x direction x type"""
    from sppark_b200 import _lib
    l = _lib.lib()
    x = loose_words(1 << lg, seed)
    for inverse in (False, True):
        for coset in (False, True):
            for order, (inp, want) in _cases(oracle, x, inverse, coset).items():
                for entry in ("compute_ntt", "sppark_b200_ntt"):
                    y = inp.copy()
                    if entry == "compute_ntt":
                        _lib.check(l.compute_ntt(0, y.ctypes.data, lg, order, int(inverse), int(coset)))
                    else:
                        _lib.check(l.sppark_b200_ntt(0, 0, y.ctypes.data, lg, order, int(inverse), int(coset)))
                    _check(y, want, entry, lg, order, inverse, coset)


@pytest.mark.parametrize("lg", [1, 2, 3, 4, 12, 19, 20, 21, 24])
def test_single_transform_loose_words(oracle, lg, monkeypatch):
    monkeypatch.delenv("SPPARK_B200_NTT_WARP", raising=False)
    monkeypatch.delenv("SPPARK_B200_NTT_BLOCK", raising=False)
    _host_entries(oracle, lg, lg)


@pytest.mark.parametrize("knob,lg", [("SPPARK_B200_NTT_WARP", 20), ("SPPARK_B200_NTT_WARP", 22),
                                     ("SPPARK_B200_NTT_BLOCK", 4), ("SPPARK_B200_NTT_BLOCK", 9),
                                     ("SPPARK_B200_NTT_BLOCK", 13)])
def test_both_pass_kernels_loose_words(oracle, knob, lg, monkeypatch):
    """each pass kernel on loose words on the other side of the size crossover too"""
    monkeypatch.delenv("SPPARK_B200_NTT_WARP", raising=False)
    monkeypatch.delenv("SPPARK_B200_NTT_BLOCK", raising=False)
    monkeypatch.setenv(knob, "1")
    _host_entries(oracle, lg, 100 + lg)


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a).view(np.int64)).cuda()


def _host(t):
    return t.cpu().numpy().view(np.uint64)


@pytest.mark.parametrize("lg", [2, 20])
def test_device_and_batched_entries_loose_words(oracle, lg):
    """ntt_dev on one row; ntt_batch (host) and ntt_batch_dev on three rows: each row must come out
    as the oracle's transform of that row alone"""
    import torch
    from sppark_b200 import ntt
    batch = 3
    x = loose_words((batch, 1 << lg), 200 + lg)
    for inverse in (False, True):
        for coset in (False, True):
            rows = [_cases(oracle, x[b], inverse, coset) for b in range(batch)]
            for order in (NN, NR, RN, RR):
                inp = np.stack([rows[b][order][0] for b in range(batch)])
                want = np.stack([rows[b][order][1] for b in range(batch)])
                ctx = (lg, order, inverse, coset)
                d = _dev(inp[0])
                ntt.ntt_dev(d, order, int(inverse), int(coset))
                torch.cuda.synchronize()
                _check(_host(d), want[0], "ntt_dev", *ctx)
                y = inp.copy()
                ntt.ntt_batch(0, y, order, int(inverse), int(coset))
                _check(y, want, "ntt_batch", *ctx)
                d = _dev(inp)
                ntt.ntt_batch_dev(d, order, int(inverse), int(coset))
                torch.cuda.synchronize()
                _check(_host(d), want, "ntt_batch_dev", *ctx)


def _lde_definition(ofn, x, lb):
    """LDE by its definition: coefficients = iNTT(x), zero-padded, coset NTT of the 2^lb-times
    larger domain"""
    c = ofn(x, NN, True, nthreads=16)
    ext = np.zeros(c.size << lb, dtype=c.dtype)
    ext[:c.size] = c
    return ofn(ext, NN, False, True, nthreads=16), c


@pytest.mark.parametrize("lg", [3, 20])
def test_lde_loose_words(oracle, lg):
    """ntt.LDE, the LDE_powers / LDE_expand device composition and lde_batch_dev"""
    import torch
    from sppark_b200 import _lib, ntt
    l = _lib.lib()
    lb = 1
    n, n_ext = 1 << lg, 1 << (lg + lb)
    x = loose_words((2, n), 300 + lg)
    defs = [_lde_definition(oracle.ntt_gl64, _reduce(x[b]), lb) for b in range(2)]
    for b, (want, coeffs) in enumerate(defs):
        ext, aux = ntt.LDE(0, x[b].copy(), lb, want_coefficients=True)
        _check(ext, want, "LDE", lg, b)
        _check(aux, coeffs, "LDE coefficients", lg, b)
        d = torch.zeros(n_ext, dtype=torch.int64, device="cuda")
        tail = d[n_ext - n:]
        tail.copy_(_dev(x[b]))
        s = torch.cuda.current_stream().cuda_stream
        _lib.check(l.sppark_b200_ntt_dev(0, tail.data_ptr(), lg, NR, 1, 0, s))
        _lib.check(l.sppark_b200_lde_powers_dev(0, tail.data_ptr(), lg, s))
        _lib.check(l.sppark_b200_lde_expand_dev(0, d.data_ptr(), tail.data_ptr(), lg, lb, s))
        _lib.check(l.sppark_b200_ntt_dev(0, d.data_ptr(), lg + lb, RN, 0, 0, s))
        torch.cuda.synchronize()
        _check(_host(d), want, "LDE_powers/LDE_expand", lg, b)
    d_in = _dev(x)
    out = ntt.lde_batch_dev(d_in, lb)
    torch.cuda.synchronize()
    r = _brev(lg)
    for b, (want, coeffs) in enumerate(defs):
        _check(_host(out)[b], want, "lde_batch_dev", lg, b)
        _check(_host(d_in)[b], coeffs[r], "lde_batch_dev coefficients", lg, b)


@pytest.mark.parametrize("lg,lg_g", [(16, 1), (20, 3)])
def test_slab_passes_loose_words(oracle, lg, lg_g):
    """the slab-sharded transform's two stages, G ranks one after another on this GPU: staging
    route (exchange as a tensor shuffle) and fused-exchange route (stores into the receivers)"""
    import torch
    from sppark_b200 import _lib, parallel
    G = 1 << lg_g
    n_local = (1 << lg) // G
    x = loose_words(1 << lg, 400 + lg)
    stream = torch.cuda.current_stream().cuda_stream
    for inverse in (False, True):
        want = oracle.ntt_gl64(_reduce(x), NN, inverse, nthreads=16)
        locs = [_dev(parallel.scatter_columns(x, lg, lg_g, r).reshape(-1)) for r in range(G)]
        staged = []
        for r in range(G):
            st = torch.empty_like(locs[r])
            parallel.gpu_slab_pass(0, lg, lg_g, r, inverse)(1, locs[r], st)
            staged.append(st.view(G, -1))
        staged = [torch.cat([staged[q][r] for q in range(G)]).contiguous() for r in range(G)]
        peers = parallel.SlabPeers(n_local * 8, nbuf=1)
        fused = [peers.tensor(0, torch.int64)] + [torch.empty(n_local, dtype=torch.int64, device="cuda")
                                                  for _ in range(G - 1)]
        ptrs = (C.c_void_p * G)(*[t.data_ptr() for t in fused])
        for r in range(G):
            _lib.check(_lib.lib().sppark_b200_ntt_slab_pass_p2p(0, locs[r].data_ptr(), ptrs, lg, lg_g, r,
                                                                int(inverse), stream))
        for route, recv in (("staging", staged), ("fused", fused)):
            scratch = torch.empty(n_local, dtype=torch.int64, device="cuda")
            for r in range(G):
                parallel.gpu_slab_pass(0, lg, lg_g, r, inverse)(2, recv[r], scratch)
            got = parallel.gather_columns([_host(t) for t in recv], lg, lg_g)
            _check(got, want, route, lg, lg_g, inverse)
        peers.close()


def test_polynomial_helpers_loose_words():
    """prefix sums / products, division by (x - z) and evaluation read loose words (and a loose z
    and loose points) as their values mod p"""
    from oracle import poly as op
    from sppark_b200 import poly
    n = 3 * 2048 + 5                                       # several scan tiles
    x = loose_words(n, 500)
    c = op.decode("gl64", x)
    y = x.copy()
    poly.prefix_op(poly.ADD, y)
    _check(y, op.encode("gl64", op.prefix_op(GL_P, "add", c)), "prefix add")
    xm = np.where(_reduce(x) == 0, np.uint64(5), x)        # no zero factor: every product stays live
    y = xm.copy()
    poly.prefix_op(poly.MULTIPLY, y)
    _check(y, op.encode("gl64", op.prefix_op(GL_P, "mul", op.decode("gl64", xm))), "prefix mul")
    z = GL_P + 12345
    for rot in (False, True):
        y = x.copy()
        poly.div_by_x_minus_z(y, np.array([z], dtype=np.uint64), rotate=rot)
        _check(y, op.encode("gl64", op.div_by_x_minus_z(GL_P, c, z % GL_P, rot)), "div_by_x_minus_z", rot)
    pts = np.array([2**64 - 1, GL_P, GL_P + 7, 3, 0], dtype=np.uint64)
    got = poly.evaluate(x, pts)
    _check(got, op.encode("gl64", op.evaluate(GL_P, c, op.decode("gl64", pts))), "evaluate")


# ---- coset transforms and LDE where the tables change level ----------------------------------

@pytest.mark.parametrize("field,lg,loose", [("gl64", 20, False), ("gl64", 25, False), ("gl64", 25, True),
                                            ("bb31", 20, False), ("bb31", 25, False)])
def test_coset_past_the_third_table(oracle, field, lg, loose):
    """coset_NTT in NN and NR, coset_iNTT in NN and RN; one oracle transform per direction.
    Canonical inputs: the inverse takes the forward oracle result and must give back x."""
    from sppark_b200 import ntt
    ofn = oracle.ntt_gl64 if field == "gl64" else oracle.ntt_bb31
    n = 1 << lg
    r = _brev(lg)
    x = loose_words(n, 600 + lg) if loose else _rand(field, n, 600 + lg)
    fwd = ofn(_reduce(x) if loose else x, NN, False, True, nthreads=16)
    for order, inp, want in ((NN, x, fwd), (NR, x, fwd[r])):
        y = inp.copy()
        ntt.coset_NTT(0, y, order)
        assert np.array_equal(y, want), (field, lg, loose, "forward", order)
    if loose:
        src = loose_words(n, 700 + lg)
        inv = ofn(_reduce(src), NN, True, True, nthreads=16)
    else:
        src, inv = fwd, x
    for order, inp in ((NN, src), (RN, np.ascontiguousarray(src[r]))):
        y = inp.copy()
        ntt.coset_iNTT(0, y, order)
        assert np.array_equal(y, inv), (field, lg, loose, "inverse", order)


def _bb_eval(a, z, lg_chunk=22):
    """sum_j a[j] * z^j mod p over BabyBear words, in chunks of 2^lg_chunk terms (products < 2^62)"""
    p = BB_P
    pw = np.ones(1, dtype=np.uint64)
    while pw.size < (1 << lg_chunk):                       # doubling: pw[m:2m] = pw[:m] * z^m
        pw = np.concatenate([pw, pw * np.uint64(pow(z, pw.size, p)) % np.uint64(p)])
    step, scale, acc = pow(z, 1 << lg_chunk, p), 1, 0
    for s in range(0, a.size, 1 << lg_chunk):
        chunk = a[s:s + (1 << lg_chunk)].astype(np.uint64)
        t = pw * np.uint64(scale) % np.uint64(p)
        acc = (acc + int((chunk * t % np.uint64(p)).sum(dtype=np.uint64))) % p
        scale = scale * step % p
    return acc


def test_babybear_coset_2pow27_field_maximum():
    """2^27, the largest BabyBear domain: a few outputs of the NR coset transform against the
    definition X[k] = sum_j x[j] (g w^k)^j (g = 3, w = 137 of order 2^27; words are Montgomery
    forms, which the linear map carries through), then the RN coset inverse gives x back"""
    from sppark_b200 import ntt
    lg = 27
    a = _rand("bb31", 1 << lg, 27)
    v = a.copy()
    ntt.coset_NTT(0, v, NR)
    for k in (0, 1, 5, (1 << 26) + 3, (1 << lg) - 1):
        pos = int(format(k, f"0{lg}b")[::-1], 2)           # NR: X[k] sits at bitrev(k)
        assert int(v[pos]) == _bb_eval(a, 3 * pow(137, k, BB_P) % BB_P), k
    ntt.coset_iNTT(0, v, RN)
    assert np.array_equal(v, a)


@pytest.mark.parametrize("field,lg,lb", [("gl64", 20, 1), ("gl64", 25, 1), ("bb31", 20, 2)])
def test_lde_past_the_third_table(oracle, field, lg, lb):
    from sppark_b200 import ntt
    ofn = oracle.ntt_gl64 if field == "gl64" else oracle.ntt_bb31
    x = _rand(field, 1 << lg, 800 + lg)
    ext, coeffs = ntt.LDE(0, x, lb, want_coefficients=True)
    want, c = _lde_definition(ofn, x, lb)
    assert np.array_equal(coeffs, c), (field, lg, lb)
    assert np.array_equal(ext, want), (field, lg, lb)
