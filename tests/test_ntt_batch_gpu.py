"""GPU: the batched NTT / LDE entry points against the single-transform entries row by row
(bit-exact), against the CPU oracle on a subset, past 2^32 elements, through the host pipeline and
on a non-default stream."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

GL_P = 2**64 - 2**32 + 1
BB_P = 0x78000001
WIDE = {2: "bls12_381_fr", 3: "vesta_fp", 4: "pallas_fp", 5: "bn254_fr", 6: "bls12_377_fr"}
NAMES = {0: "gl64", 1: "bb31", **WIDE}


def _host(field, batch, lg, seed):
    rng = np.random.default_rng(seed)
    if field == 0:
        return rng.integers(0, GL_P, size=(batch, 1 << lg), dtype=np.uint64)
    if field == 1:
        return rng.integers(0, BB_P, size=(batch, 1 << lg), dtype=np.uint32)
    a = rng.integers(0, 2**63, size=(batch, 1 << lg, 4), dtype=np.uint64)
    a[..., 3] >>= np.uint64(4)              # < 2^252: below every 256-bit modulus here
    return a


def _dev(a):
    import torch
    return torch.from_numpy(a.view(np.int64 if a.dtype == np.uint64 else np.int32)).cuda()


def _single_rows(field, d, lg, order, direction, typ):
    """the single-transform entry on every row of d (in place)"""
    import torch
    from sppark_b200 import _lib
    s = torch.cuda.current_stream().cuda_stream
    row = d[0].numel() * d.element_size()
    for b in range(d.shape[0]):
        _lib.check(_lib.lib().sppark_b200_ntt_dev(field, d.data_ptr() + b * row, lg, order, direction, typ, s))


def _parity(field, lg, batch, seed, combos=None):
    import torch
    from sppark_b200 import ntt
    x = _dev(_host(field, batch, lg, seed))
    for order in range(5):
        for direction in (0, 1):
            for typ in (0, 1):
                if combos is not None and (order, direction, typ) not in combos:
                    continue
                got, want = x.clone(), x.clone()
                ntt.ntt_batch_dev(got, order, direction, typ, field=field)
                _single_rows(field, want, lg, order, direction, typ)
                torch.cuda.synchronize()
                assert torch.equal(got, want), (NAMES[field], lg, batch, order, direction, typ)


ALL = None
SOME = {(0, 0, 0), (1, 1, 0), (2, 0, 1), (3, 1, 1), (4, 0, 0), (4, 1, 1)}


@pytest.mark.parametrize("field", [0, 1])
@pytest.mark.parametrize("lg", [1, 2, 3, 4, 5, 6, 8, 9, 10, 12, 13, 16, 17, 19, 20, 21])
def test_row_parity_single_word(field, lg, monkeypatch):
    """lg 4..19 take the warp path, 1..3 and 20+ the block path"""
    monkeypatch.delenv("SPPARK_B200_NTT_WARP", raising=False)
    monkeypatch.delenv("SPPARK_B200_NTT_BLOCK", raising=False)
    for batch in (1, 3, 7, 64):
        if batch << lg <= 1 << 24:
            _parity(field, lg, batch, 100 * lg + batch, ALL if batch != 64 or lg <= 12 else SOME)
    if lg <= 10:
        _parity(field, lg, 1000, lg, SOME)


@pytest.mark.parametrize("path", ["SPPARK_B200_NTT_WARP", "SPPARK_B200_NTT_BLOCK"])
@pytest.mark.parametrize("field", [0, 1])
def test_row_parity_forced_path(field, path, monkeypatch):
    monkeypatch.delenv("SPPARK_B200_NTT_WARP", raising=False)
    monkeypatch.delenv("SPPARK_B200_NTT_BLOCK", raising=False)
    monkeypatch.setenv(path, "1")
    for lg, batch in ((4, 7), (8, 3), (8, 64), (9, 1000), (12, 7), (16, 3), (20, 3), (21, 3)):
        _parity(field, lg, batch, lg + batch, ALL if batch < 64 else SOME)


@pytest.mark.parametrize("field", [2, 3, 4, 5, 6])
def test_row_parity_256bit(field):
    for lg, batch in ((1, 7), (3, 3), (4, 1000), (8, 64), (11, 3), (12, 7), (14, 3)):
        _parity(field, lg, batch, field * 100 + lg, ALL if batch < 64 else SOME)


def test_batch_matches_oracle(oracle):
    """independently of the single-transform path: rows against the CPU oracle"""
    import torch
    from sppark_b200 import ntt
    for field, lg, batch in ((0, 10, 3), (1, 13, 3), (0, 20, 2), (2, 6, 3)):
        x = _host(field, batch, lg, lg)
        if field == 0:
            ofn = lambda a, *k: oracle.ntt_gl64(a, *k, nthreads=8)        # noqa: E731
        elif field == 1:
            ofn = lambda a, *k: oracle.ntt_bb31(a, *k, nthreads=8)        # noqa: E731
        else:
            ofn = lambda a, *k: oracle.ntt_ff(WIDE[field], a, *k)         # noqa: E731
        for order in range(4):
            for direction in (0, 1):
                for typ in (0, 1):
                    d = _dev(x)
                    ntt.ntt_batch_dev(d, order, direction, typ, field=field)
                    got = d.cpu().numpy().view(x.dtype)
                    for b in range(batch):
                        want = ofn(x[b], order, bool(direction), bool(typ))
                        assert np.array_equal(got[b], want.reshape(got[b].shape)), (field, lg, order, direction, typ, b)


@pytest.mark.parametrize("lg", [20, 16])
def test_offsets_past_2pow32_elements(lg):
    """bb31, NR in place over 2^32 + 2^lg elements (16 GiB + one row): lg 20 takes the block path,
    lg 16 the warp path; the rows on both sides of element 2^32 must match the single transform"""
    import torch
    from sppark_b200 import ntt
    batch = (1 << (32 - lg)) + 1
    need = (batch << lg) * 4
    if torch.cuda.mem_get_info()[0] < need + (1 << 30):
        pytest.skip("not enough free device memory")
    g = torch.Generator(device="cuda")
    g.manual_seed(lg)
    d = torch.randint(0, BB_P, (batch, 1 << lg), dtype=torch.int32, device="cuda", generator=g)
    rows = [0, batch // 2, (1 << (32 - lg)) - 1, 1 << (32 - lg)]
    before = d[rows].clone()
    ntt.ntt_batch_dev(d, ntt.NR, ntt.FORWARD, ntt.STANDARD, field=ntt.BB31)
    _single_rows(1, before, lg, ntt.NR, 0, 0)
    torch.cuda.synchronize()
    assert torch.equal(d[rows], before)
    del d
    torch.cuda.empty_cache()


@pytest.mark.parametrize("field", [0, 1, 2, 5])
def test_lde_batch(oracle, field):
    import torch
    from sppark_b200 import _lib, ntt
    for lg, lb, batch in ((5, 1, 3), (12, 2, 3), (17, 1, 2)):
        if field >= 2 and lg > 12:
            continue
        x = _host(field, batch, lg, 7 * lg + lb)
        d_in = _dev(x)
        ext = ntt.lde_batch_dev(d_in, lb, field=field)
        torch.cuda.synchronize()
        got_ext = ext.cpu().numpy().view(x.dtype)
        got_coef = d_in.cpu().numpy().view(x.dtype)
        idx = np.array([int(format(i, f"0{lg}b")[::-1], 2) for i in range(1 << lg)])
        for b in range(batch):
            one = np.zeros((x.shape[1] << lb,) + x.shape[2:], dtype=x.dtype)
            one[:x.shape[1]] = x[b]
            aux = np.zeros_like(x[b])
            _lib.check(_lib.lib().sppark_b200_lde(field, 0, one.ctypes.data, lg, lb, aux.ctypes.data))
            assert np.array_equal(got_ext[b], one), (field, lg, b)
            assert np.array_equal(got_coef[b], aux[idx]), (field, lg, b)      # bit-reversed coefficients
            if b == 0 and lg <= 12:
                want, _ = oracle.lde(NAMES[field], x[b], lb)
                assert np.array_equal(got_ext[b], want.reshape(got_ext[b].shape)), (field, lg)


def test_lde_batch_arguments():
    """lg 0 and batch 0 are no-ops; a wrapping lg_blowup and overlapping buffers are rejected before
    any work, leaving both buffers as they were"""
    import torch
    from sppark_b200 import _lib
    l = _lib.lib()
    s = torch.cuda.current_stream().cuda_stream
    buf = torch.arange(64, dtype=torch.int64, device="cuda")
    before = buf.clone()
    assert l.sppark_b200_lde_batch_dev(0, buf.data_ptr() + 256, buf.data_ptr(), 0, 1, 4, s).code == 0
    assert l.sppark_b200_lde_batch_dev(0, buf.data_ptr() + 256, buf.data_ptr(), 3, 1, 0, s).code == 0
    for args in ((0, buf.data_ptr() + 256, buf.data_ptr(), 3, 0xFFFFFFFE, 1, s),   # lg + lg_blowup wraps
                 (0, buf.data_ptr() + 64, buf.data_ptr(), 3, 1, 2, s),             # d_out overlaps d_in
                 (0, buf.data_ptr(), buf.data_ptr() + 128, 3, 1, 2, s)):           # d_in inside d_out
        e = l.sppark_b200_lde_batch_dev(*args)
        assert e.code != 0, args
        if e.message:
            l.drop_error_message(e.message)
    torch.cuda.synchronize()
    assert torch.equal(buf, before)


@pytest.mark.parametrize("lg,batch", [(20, 11), (22, 5), (9, 3000)])
def test_host_entry_matches_device_entry(lg, batch):
    """several pipeline groups with a short tail, from a pinned torch buffer and a pageable numpy one"""
    import torch
    from sppark_b200 import ntt
    x = _host(0, batch, lg, lg)
    for order, direction, typ in ((ntt.NN, 0, 0), (ntt.RN, 1, 1)):
        d = _dev(x)
        ntt.ntt_batch_dev(d, order, direction, typ)
        want = d.cpu().numpy().view(np.uint64)
        pinned = torch.from_numpy(x.view(np.int64)).pin_memory()
        ntt.ntt_batch(0, pinned.numpy().view(np.uint64), order, direction, typ)
        assert np.array_equal(pinned.numpy().view(np.uint64), want), ("pinned", order)
        pageable = x.copy()
        ntt.ntt_batch(0, pageable, order, direction, typ)
        assert np.array_equal(pageable, want), ("pageable", order)


def test_host_entry_invalid_arguments_leave_buffer():
    from sppark_b200 import _lib
    l = _lib.lib()
    buf = _host(1, 3, 8, 1)
    before = buf.copy()
    for args in ((1, 0, buf.ctypes.data, 8, 3, 5, 0, 0),            # order out of range
                 (1, 0, buf.ctypes.data, 28, 3, 0, 0, 0),           # 2^28 BabyBear does not exist
                 (0, 0, buf.ctypes.data, 30, 1 << 40, 0, 0, 0),     # byte size overflows size_t
                 (9, 0, buf.ctypes.data, 8, 3, 0, 0, 0)):           # unknown field
        e = l.sppark_b200_ntt_batch(*args)
        assert e.code != 0, args
        if e.message:
            l.drop_error_message(e.message)
        assert np.array_equal(buf, before), args
    assert l.sppark_b200_ntt_batch(1, 0, buf.ctypes.data, 8, 0, 0, 0, 0).code == 0   # batch 0: no-op
    assert l.sppark_b200_ntt_batch(1, 0, buf.ctypes.data, 0, 3, 0, 0, 0).code == 0   # lg 0: no-op
    assert np.array_equal(buf, before)


def test_device_entries_on_side_stream():
    """enqueued on a non-default torch stream, ordered before work queued after them there"""
    import torch
    from sppark_b200 import ntt
    x = _host(0, 16, 16, 3)
    want = _dev(x)
    ntt.ntt_batch_dev(want, ntt.NR)
    want_lde = ntt.lde_batch_dev(_dev(x), 1)
    torch.cuda.synchronize()
    src = torch.from_numpy(x.view(np.int64)).pin_memory()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        d = torch.empty(src.shape, dtype=src.dtype, device="cuda")
        d.copy_(src, non_blocking=True)
        ntt.ntt_batch_dev(d, ntt.NR)
        after = d.clone()                      # queued after the transform on the same stream
        d2 = torch.empty_like(d)
        d2.copy_(src, non_blocking=True)
        ext = ntt.lde_batch_dev(d2, 1)
        ext_after = ext.clone()
    side.synchronize()
    assert torch.equal(after, want)
    assert torch.equal(ext_after, want_lde)
