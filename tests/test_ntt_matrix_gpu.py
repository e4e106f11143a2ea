"""GPU: NTT and LDE down the columns of a row-major matrix against the batched entries on the
transposed matrix (what a caller does without the matrix entries), bit-exactly: every order,
direction and type, widths below, at and across the column block, Goldilocks loose words, more than
2^32 elements, the host entry on pinned and pageable memory, a non-default stream and the refusals."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

GL_P = 2**64 - 2**32 + 1
BB_P = 0x78000001
ALL = [(o, d, t) for o in range(5) for d in (0, 1) for t in (0, 1)]
SOME = [(0, 0, 0), (1, 1, 0), (2, 0, 1), (3, 1, 1), (4, 0, 0), (4, 1, 1)]
WIDTHS = [1, 3, 4, 8, 13, 64, 100, 256]


def _host(field, lg, width, seed):
    rng = np.random.default_rng(seed)
    if field == 0:
        return rng.integers(0, GL_P, size=(1 << lg, width), dtype=np.uint64)
    return rng.integers(0, BB_P, size=(1 << lg, width), dtype=np.uint32)


def _dev(a):
    import torch
    return torch.from_numpy(a.view(np.int64 if a.dtype == np.uint64 else np.int32)).cuda()


def _via_transpose(d, order, direction, typ, field):
    """transpose -> ntt_batch_dev -> transpose back"""
    from sppark_b200 import ntt
    t = d.t().contiguous()
    ntt.ntt_batch_dev(t, order, direction, typ, field=field)
    return t.t().contiguous()


def _parity(field, x, combos):
    import torch
    from sppark_b200 import ntt
    d = _dev(x)
    lg = x.shape[0].bit_length() - 1
    for order, direction, typ in combos:
        got = d.clone()
        ntt.ntt_matrix_dev(got, order, direction, typ, field=field)
        want = _via_transpose(d, order, direction, typ, field)
        torch.cuda.synchronize()
        assert torch.equal(got, want), (field, lg, x.shape[1], order, direction, typ)


@pytest.mark.parametrize("lg", [1, 2, 3, 4, 5, 6, 8, 10, 12, 13, 16, 19, 20, 21])
@pytest.mark.parametrize("field", [0, 1])
def test_matrix_matches_transposed_batch(field, lg):
    """all orders, directions and types; widths capped at 2^24 elements (2^22 for all 20 combinations)"""
    for width in WIDTHS:
        if width << lg > 1 << 24:
            continue
        combos = ALL if width << lg <= 1 << 22 else SOME
        _parity(field, _host(field, lg, width, 1000 * field + 10 * lg + width), combos)


@pytest.mark.parametrize("field", [0, 1])
def test_matrix_2pow24(field):
    _parity(field, _host(field, 24, 3, 24 + field), SOME)


@pytest.mark.parametrize("field", [0, 1])
def test_width_one_equals_ntt_dev(field):
    import torch
    from sppark_b200 import ntt
    for lg in (3, 11, 20):
        x = _host(field, lg, 1, lg)
        for order, direction, typ in ALL:
            got, want = _dev(x), _dev(x.reshape(-1))
            ntt.ntt_matrix_dev(got, order, direction, typ, field=field)
            ntt.ntt_dev(want, order, direction, typ, field=field)
            torch.cuda.synchronize()
            assert torch.equal(got.reshape(-1), want), (field, lg, order, direction, typ)


@pytest.mark.parametrize("field", [0, 1])
def test_lde_matrix_matches_lde_batch(field):
    """d_out against lde_batch_dev on the transposed input, and the coefficients left in d_in"""
    import torch
    from sppark_b200 import ntt
    for lg, width in ((1, 3), (5, 13), (12, 4), (17, 9), (20, 5)):
        for lb in (1, 2, 3):
            x = _host(field, lg, width, 7 * lg + lb)
            d_in = _dev(x)
            ext = ntt.lde_matrix_dev(d_in, lb, field=field)
            t_in = _dev(np.ascontiguousarray(x.T))
            t_ext = ntt.lde_batch_dev(t_in, lb, field=field)
            torch.cuda.synchronize()
            assert ext.shape == ((1 << lg) << lb, width)
            assert torch.equal(ext, t_ext.t()), (field, lg, width, lb)
            assert torch.equal(d_in, t_in.t()), (field, lg, width, lb)


def test_goldilocks_loose_words():
    """any uint64 is a Goldilocks input word (its value mod p): the matrix result equals the
    transposed batch on the same words, and the oracle-checked batch on the reduced words"""
    import torch
    from sppark_b200 import ntt
    rng = np.random.default_rng(5)
    for lg, width in ((3, 5), (12, 9), (20, 4), (21, 3)):
        n = (1 << lg) * width
        high = np.uint64(GL_P) + rng.integers(0, 2**32 - 1, size=n, dtype=np.uint64)
        low = rng.integers(0, 2**32, size=n, dtype=np.uint64)
        x = np.choose(rng.integers(0, 2, size=n), [high, low]).reshape(1 << lg, width)
        reduced = np.where(x >= np.uint64(GL_P), x - np.uint64(GL_P), x)
        for order, direction, typ in SOME:
            got = _dev(x)
            ntt.ntt_matrix_dev(got, order, direction, typ, field=0)
            want = _via_transpose(_dev(reduced), order, direction, typ, 0)
            torch.cuda.synchronize()
            assert torch.equal(got, want), (lg, width, order, direction, typ)
        d_in = _dev(x)
        ext = ntt.lde_matrix_dev(d_in, 1, field=0)
        t_ext = ntt.lde_batch_dev(_dev(np.ascontiguousarray(reduced.T)), 1, field=0)
        torch.cuda.synchronize()
        assert torch.equal(ext, t_ext.t()), (lg, width)


@pytest.mark.parametrize("lg,width", [(20, 9), (12, 100)])
def test_host_entry_pinned_and_pageable(lg, width):
    import torch
    from sppark_b200 import ntt
    x = _host(0, lg, width, lg)
    for order, direction, typ in ((0, 0, 0), (2, 1, 1), (4, 0, 1)):
        d = _dev(x)
        ntt.ntt_matrix_dev(d, order, direction, typ)
        want = d.cpu().numpy().view(np.uint64)
        pinned = torch.from_numpy(x.view(np.int64)).pin_memory()
        ntt.ntt_matrix(0, pinned.numpy().view(np.uint64), order, direction, typ)
        assert np.array_equal(pinned.numpy().view(np.uint64), want), ("pinned", order)
        pageable = x.copy()
        ntt.ntt_matrix(0, pageable, order, direction, typ)
        assert np.array_equal(pageable, want), ("pageable", order)
    xb = _host(1, 10, 7, 3)
    d = _dev(xb)
    ntt.ntt_matrix_dev(d, 1, 0, 0)
    hb = xb.copy()
    ntt.ntt_matrix(0, hb, 1, 0, 0)
    assert np.array_equal(hb, d.cpu().numpy().view(np.uint32))


def test_device_entries_on_side_stream():
    """enqueued on a non-default torch stream, ordered before work queued after them there"""
    import torch
    from sppark_b200 import ntt
    x = _host(0, 16, 24, 3)
    want = _dev(x)
    ntt.ntt_matrix_dev(want, ntt.NN)
    want_lde = ntt.lde_matrix_dev(_dev(x), 1)
    torch.cuda.synchronize()
    src = torch.from_numpy(x.view(np.int64)).pin_memory()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        d = torch.empty(src.shape, dtype=src.dtype, device="cuda")
        d.copy_(src, non_blocking=True)
        ntt.ntt_matrix_dev(d, ntt.NN)
        after = d.clone()
        d2 = torch.empty_like(d)
        d2.copy_(src, non_blocking=True)
        ext = ntt.lde_matrix_dev(d2, 1)
        ext_after = ext.clone()
    side.synchronize()
    assert torch.equal(after, want)
    assert torch.equal(ext_after, want_lde)


def test_past_2pow32_elements():
    """BabyBear 2^24 x 260 (2^32 + 2^26 elements, 17 GiB), NR in place: a seeded sample of columns,
    among them the last, against ntt_batch_dev of those columns"""
    import torch
    from sppark_b200 import ntt
    lg, width = 24, 260
    need = (width << lg) * 4
    if torch.cuda.mem_get_info()[0] < need + (4 << 30):
        pytest.skip("not enough free device memory")
    g = torch.Generator(device="cuda")
    g.manual_seed(24)
    d = torch.randint(0, BB_P, (1 << lg, width), dtype=torch.int32, device="cuda", generator=g)
    cols = sorted(set(np.random.default_rng(1).choice(width, 5, replace=False).tolist()) | {0, width - 1})
    sample = d[:, cols].t().contiguous()
    ntt.ntt_matrix_dev(d, ntt.NR, ntt.FORWARD, ntt.STANDARD, field=ntt.BB31)
    ntt.ntt_batch_dev(sample, ntt.NR, ntt.FORWARD, ntt.STANDARD, field=ntt.BB31)
    torch.cuda.synchronize()
    assert torch.equal(d[:, cols].t(), sample)
    del d, sample
    torch.cuda.empty_cache()


def test_refusals_leave_memory():
    """256-bit fields, overlapping LDE buffers and out-of-range lg are -cudaErrorInvalidValue, before
    any work; lg 0 and width 0 are no-ops"""
    import ctypes as C
    import torch
    from sppark_b200 import _lib, ntt
    l = _lib.lib()
    s = torch.cuda.current_stream().cuda_stream
    buf = torch.arange(8 * 64, dtype=torch.int64, device="cuda")
    before = buf.clone()
    p = buf.data_ptr()
    cases = [l.sppark_b200_ntt_matrix_dev(2, p, 3, 4, 0, 0, 0, s),                  # BLS12-381 Fr
             l.sppark_b200_lde_matrix_dev(3, p + 2048, p, 3, 1, 4, s),              # Pallas
             l.sppark_b200_lde_matrix_dev(0, p + 64, p, 3, 1, 4, s),                # d_out overlaps d_in
             l.sppark_b200_lde_matrix_dev(0, p, p + 128, 3, 1, 4, s),               # d_in inside d_out
             l.sppark_b200_lde_matrix_dev(0, p + 2048, p, 3, 0xFFFFFFFE, 4, s),     # lg + lg_blowup wraps
             l.sppark_b200_lde_matrix_dev(1, p + 2048, p, 26, 2, 1, s),             # 2^28 BabyBear
             l.sppark_b200_ntt_matrix_dev(0, p, 33, 1, 0, 0, 0, s),                 # 2^33 Goldilocks
             l.sppark_b200_ntt_matrix_dev(1, p, 28, 1, 0, 0, 0, s)]                 # 2^28 BabyBear
    for e in cases:
        assert e.code == -1
        msg = C.cast(e.message, C.c_char_p).value.decode() if e.message else ""
        if e.message:
            l.drop_error_message(e.message)
        assert msg
    assert l.sppark_b200_ntt_matrix_dev(0, p, 0, 4, 0, 0, 0, s).code == 0
    assert l.sppark_b200_ntt_matrix_dev(0, p, 3, 0, 0, 0, 0, s).code == 0
    assert l.sppark_b200_lde_matrix_dev(0, p + 2048, p, 3, 1, 0, s).code == 0
    torch.cuda.synchronize()
    assert torch.equal(buf, before)
    with pytest.raises(ValueError):
        ntt.ntt_matrix_dev(buf.view(8, 64), field=ntt.BLS12_381_FR)
    with pytest.raises(ValueError):
        ntt.ntt_matrix_dev(buf.view(8, 64).int(), field=ntt.GL64)     # 4-byte words, 8-byte field
    with pytest.raises(ValueError):
        ntt.ntt_matrix_dev(buf.view(2, 4, 64))                         # rank 3
    assert torch.equal(buf, before)
