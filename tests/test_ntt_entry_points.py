"""The refusals of the NTT, LDE, polynomial and word-selftest C entry points, without a GPU: for
every entry, what an unknown field id, a bad order / direction / type, a bad pass or op, or a null
argument returns -- the code and the exact message -- and which refusals come before the device is
looked for (-cudaErrorInvalidValue, -1, on any host) and which after it (-cudaErrorNoDevice, -100,
on a host without a GPU).  After every refusal the caller's buffers are as they were."""
import ctypes as C

import numpy as np
import pytest

INVAL, NODEV = -1, -100
UNKNOWN = (7, 9, -1)          # ids of no field
WIDE = (2, 3, 4, 5, 6)        # the 256-bit fields (SPPARK_FIELD_BLS12_381_FR .. SPPARK_FIELD_BLS12_377_FR)
MATRIX_WIDE = ": the matrix entries serve Goldilocks and BabyBear only, not the 256-bit fields"


def _no_gpu():
    import torch
    return not torch.cuda.is_available()


class Bufs:
    """host buffers handed to the entries as data, output, peer and z pointers"""

    def __init__(self):
        self.a = np.arange(1, 1 + 8 * 64, dtype=np.uint64)
        self.b = np.arange(1000, 1000 + 8 * 64, dtype=np.uint64)
        self.ids = np.zeros(4, dtype=np.int32)
        self.keep = (self.a.copy(), self.b.copy(), self.ids.copy())

    def unchanged(self):
        return all(np.array_equal(x, y) for x, y in zip((self.a, self.b, self.ids), self.keep))


def _call(lib, name, *args):
    e = getattr(lib, name)(*args)
    msg = C.cast(e.message, C.c_char_p).value.decode() if e.message else None
    if e.message:
        lib.drop_error_message(e.message)
    return e.code, msg


# entry -> (args of a call that the field id alone decides, as a function of (field, buffers)).
# Well-formed otherwise: lg 3, batch / width 2, order NN, forward, standard.
def _entries(u):
    a, b = u.a.ctypes.data, u.b.ctypes.data
    return {
        "sppark_b200_ntt": lambda f: (f, 0, a, 3, 0, 0, 0),
        "sppark_b200_ntt_dev": lambda f: (f, a, 3, 0, 0, 0, None),
        "sppark_b200_lde": lambda f: (f, 0, a, 3, 1, None),
        "sppark_b200_lde_powers_dev": lambda f: (f, a, 3, None),
        "sppark_b200_lde_expand_dev": lambda f: (f, b, a, 3, 1, None),
        "sppark_b200_ntt_batch_dev": lambda f: (f, a, 3, 2, 0, 0, 0, None),
        "sppark_b200_lde_batch_dev": lambda f: (f, b, a, 3, 1, 2, None),
        "sppark_b200_ntt_batch": lambda f: (f, 0, a, 3, 2, 0, 0, 0),
        "sppark_b200_ntt_slab_pass": lambda f: (f, 1, a, b, 4, 1, 0, 0, None),
        "sppark_b200_ntt_slab_pass_p2p": lambda f: (f, a, u.ids.ctypes.data, 4, 1, 0, 0, None),
        "sppark_b200_ntt_matrix_dev": lambda f: (f, a, 3, 2, 0, 0, 0, None),
        "sppark_b200_lde_matrix_dev": lambda f: (f, b, a, 3, 1, 2, None),
        "sppark_b200_ntt_matrix": lambda f: (f, 0, a, 3, 2, 0, 0, 0),
        "sppark_b200_prefix_op_dev": lambda f: (f, 0, b, a, 16, None),
        "sppark_b200_div_by_x_minus_z_dev": lambda f: (f, a, 16, b, 0, None),
        "sppark_b200_evaluate_dev": lambda f: (f, b, a, 2, a, 16, None),
        "sppark_b200_batch_inverse_dev": lambda f: (f, b, a, 16, None),
        "sppark_b200_selftest_word_field": lambda f: (f, 1, 16, b, a, a),
    }


UNKNOWN_FIELD_MSG = {
    "sppark_b200_ntt": "sppark_b200_ntt: unknown field",
    "sppark_b200_ntt_dev": "sppark_b200_ntt_dev: unknown field",
    "sppark_b200_lde": "sppark_b200_lde: unknown field",
    "sppark_b200_lde_powers_dev": "sppark_b200_lde_*_dev: unknown field",
    "sppark_b200_lde_expand_dev": "sppark_b200_lde_*_dev: unknown field",
    "sppark_b200_ntt_batch_dev": "sppark_b200_ntt_batch_dev: unknown field",
    "sppark_b200_lde_batch_dev": "sppark_b200_lde_batch_dev: unknown field",
    "sppark_b200_ntt_batch": "sppark_b200_ntt_batch: unknown field",
    "sppark_b200_ntt_slab_pass": "sppark_b200_ntt_slab_pass: unknown field",
    "sppark_b200_ntt_slab_pass_p2p": "sppark_b200_ntt_slab_pass_p2p: unknown field",
    "sppark_b200_ntt_matrix_dev": "sppark_b200_ntt_matrix_dev: unknown field",
    "sppark_b200_lde_matrix_dev": "sppark_b200_lde_matrix_dev: unknown field",
    "sppark_b200_ntt_matrix": "sppark_b200_ntt_matrix: unknown field",
    "sppark_b200_prefix_op_dev": "sppark_b200 polynomial: unknown field",
    "sppark_b200_div_by_x_minus_z_dev": "sppark_b200 polynomial: unknown field",
    "sppark_b200_evaluate_dev": "sppark_b200 polynomial: unknown field",
    "sppark_b200_batch_inverse_dev": "sppark_b200 polynomial: unknown field",
    "sppark_b200_selftest_word_field": "selftest_word_field: unknown field",
}


@pytest.mark.parametrize("name", sorted(UNKNOWN_FIELD_MSG))
def test_unknown_field(lib, name):
    u = Bufs()
    args = _entries(u)[name]
    for f in UNKNOWN:
        assert _call(lib, name, *args(f)) == (INVAL, UNKNOWN_FIELD_MSG[name]), f
    assert u.unchanged()


@pytest.mark.parametrize("name", ["sppark_b200_ntt_matrix_dev", "sppark_b200_lde_matrix_dev", "sppark_b200_ntt_matrix"])
def test_matrix_entries_refuse_the_256bit_fields(lib, name):
    u = Bufs()
    args = _entries(u)[name]
    for f in WIDE:
        assert _call(lib, name, *args(f)) == (INVAL, name + MATRIX_WIDE), f
    assert u.unchanged()


def test_word_selftest_refuses_the_256bit_fields(lib):
    u = Bufs()
    args = _entries(u)["sppark_b200_selftest_word_field"]
    for f in WIDE:
        assert _call(lib, "sppark_b200_selftest_word_field", *args(f)) == (INVAL, "selftest_word_field: unknown field")
    assert u.unchanged()


# (order, direction, type) triples with one value out of range
BAD_ODT = [(5, 0, 0), (-1, 0, 0), (0, 2, 0), (0, -1, 0), (0, 0, 2), (0, 0, -1)]


def test_bad_order_direction_type(lib):
    u = Bufs()
    a = u.a.ctypes.data
    for o, d, t in BAD_ODT:
        for f in (0, 1):
            assert _call(lib, "sppark_b200_ntt", f, 0, a, 3, o, d, t) == (INVAL, "compute_ntt: bad order/direction/type")
            assert _call(lib, "sppark_b200_ntt_dev", f, a, 3, o, d, t, None) == (INVAL, "ntt_dev: bad order/direction/type")
            assert _call(lib, "sppark_b200_ntt_batch", f, 0, a, 3, 2, o, d, t) == (INVAL, "ntt_batch: bad order/direction/type")
            assert (_call(lib, "sppark_b200_ntt_batch_dev", f, a, 3, 2, o, d, t, None)
                    == (INVAL, "ntt_batch_dev: bad order/direction/type"))
            assert _call(lib, "sppark_b200_ntt_matrix", f, 0, a, 3, 2, o, d, t) == (INVAL, "ntt_matrix: bad order/direction/type")
            assert (_call(lib, "sppark_b200_ntt_matrix_dev", f, a, 3, 2, o, d, t, None)
                    == (INVAL, "ntt_matrix_dev: bad order/direction/type"))
        assert _call(lib, "compute_ntt", 0, a, 3, o, d, t) == (INVAL, "compute_ntt: bad order/direction/type")
        # a 256-bit field takes the same check
        assert _call(lib, "sppark_b200_ntt", 2, 0, a, 3, o, d, t) == (INVAL, "compute_ntt: bad order/direction/type")
    assert u.unchanged()


def test_range_checks_before_the_device(lib):
    """out-of-range sizes that the device entries refuse before looking for a device"""
    u = Bufs()
    a = u.a.ctypes.data
    assert (_call(lib, "sppark_b200_ntt_batch_dev", 1, a, 28, 1, 0, 0, 0, None)
            == (INVAL, "ntt_batch_dev: lg_domain_size or batch out of range for this field"))
    assert (_call(lib, "sppark_b200_ntt_matrix_dev", 1, a, 28, 1, 0, 0, 0, None)
            == (INVAL, "ntt_matrix_dev: lg_domain_size or width out of range for this field"))
    assert (_call(lib, "sppark_b200_ntt_matrix", 1, 0, a, 28, 1, 0, 0, 0)
            == (INVAL, "ntt_matrix: lg_domain_size or width out of range for this field"))
    assert (_call(lib, "sppark_b200_ntt_matrix", 0, 0, a, 30, 1 << 40, 0, 0, 0)
            == (INVAL, "ntt_matrix: lg_domain_size or width out of range for this field"))
    # lg 0 or width 0: a no-op that succeeds without a device
    assert _call(lib, "sppark_b200_ntt_matrix", 0, 0, a, 0, 2, 0, 0, 0) == (0, None)
    assert _call(lib, "sppark_b200_ntt_matrix", 1, 0, a, 3, 0, 0, 0, 0) == (0, None)
    assert u.unchanged()


def test_slab_pass_bad_pass_or_direction(lib):
    u = Bufs()
    a, b, peers = u.a.ctypes.data, u.b.ctypes.data, u.ids.ctypes.data
    msg = "ntt_slab_pass: bad direction / pass"
    for f in (0, 1, 2):
        for which in (0, 3, -1):
            assert _call(lib, "sppark_b200_ntt_slab_pass", f, which, a, b, 4, 1, 0, 0, None) == (INVAL, msg)
        for d in (2, -1):
            assert _call(lib, "sppark_b200_ntt_slab_pass", f, 1, a, b, 4, 1, 0, d, None) == (INVAL, msg)
            assert _call(lib, "sppark_b200_ntt_slab_pass_p2p", f, a, peers, 4, 1, 0, d, None) == (INVAL, msg)
    assert u.unchanged()


def test_slab_pass_p2p_null_peers_before_field(lib):
    u = Bufs()
    a = u.a.ctypes.data
    for f in (0, 1, 2) + UNKNOWN:
        assert (_call(lib, "sppark_b200_ntt_slab_pass_p2p", f, a, None, 4, 1, 0, 0, None)
                == (INVAL, "ntt_slab_pass_p2p: no peer buffers"))
    assert u.unchanged()


def test_sharded_null_arguments(lib):
    u = Bufs()
    a, ids = u.a.ctypes.data, u.ids.ctypes.data
    for f in (0, 1) + UNKNOWN:
        assert _call(lib, "sppark_b200_ntt_sharded", f, None, 4, 0, ids, 1) == (INVAL, "ntt_sharded: null argument")
        assert _call(lib, "sppark_b200_ntt_sharded", f, a, 4, 0, None, 1) == (INVAL, "ntt_sharded: null argument")
    assert u.unchanged()


def test_polynomial_op_and_z_before_field(lib):
    u = Bufs()
    a, b = u.a.ctypes.data, u.b.ctypes.data
    for f in (0, 2) + UNKNOWN:
        for op in (2, -1):
            assert (_call(lib, "sppark_b200_prefix_op_dev", f, op, b, a, 16, None)
                    == (INVAL, "sppark_b200_prefix_op_dev: op is 0 (add) or 1 (multiply)"))
        assert (_call(lib, "sppark_b200_div_by_x_minus_z_dev", f, a, 16, None, 0, None)
                == (INVAL, "sppark_b200_div_by_x_minus_z_dev: z is null"))
    assert u.unchanged()


# ---- refusals that come after the device lookup: -cudaErrorNoDevice on a host without a GPU ----
def _after_device_calls(u):
    a, b, ids = u.a.ctypes.data, u.b.ctypes.data, u.ids.ctypes.data
    calls = [
        ("compute_ntt", (0, a, 0, 0, 0, 0)),                                 # lg 0: select_gpu runs first
        ("sppark_b200_ntt_batch", (1, 0, a, 28, 1, 0, 0, 0)),                # lg past BabyBear's domain
        ("sppark_b200_ntt_batch", (0, 0, a, 31, 1, 0, 0, 0)),
        ("sppark_b200_lde", (0, 0, a, 0, 1, None)),                          # lg 0
        ("sppark_b200_lde", (1, 0, a, 27, 1, None)),                         # lg + lg_blowup past the domain
        ("sppark_b200_ntt_sharded", (9, a, 4, 0, ids, 1)),                   # the field is checked last
        ("sppark_b200_ntt_sharded", (-1, a, 4, 0, ids, 1)),
        ("sppark_b200_ntt_sharded", (0, a, 4, 2, ids, 1)),                   # bad direction
    ]
    # well-formed calls of every field reach the device lookup
    for f in range(7):
        calls += [("sppark_b200_ntt", (f, 0, a, 3, 0, 0, 0)), ("sppark_b200_ntt_dev", (f, a, 3, 0, 0, 0, None)),
                  ("sppark_b200_lde", (f, 0, a, 3, 1, None)), ("sppark_b200_lde_powers_dev", (f, a, 3, None)),
                  ("sppark_b200_lde_expand_dev", (f, b, a, 3, 1, None)),
                  ("sppark_b200_ntt_batch_dev", (f, a, 3, 2, 0, 0, 0, None)),
                  ("sppark_b200_lde_batch_dev", (f, b, a, 3, 1, 2, None)),
                  ("sppark_b200_ntt_batch", (f, 0, a, 3, 2, 0, 0, 0)),
                  ("sppark_b200_ntt_slab_pass", (f, 1, a, b, 4, 1, 0, 0, None)),
                  ("sppark_b200_ntt_slab_pass_p2p", (f, a, ids, 4, 1, 0, 0, None)),
                  ("sppark_b200_prefix_op_dev", (f, 1, b, a, 16, None)),
                  ("sppark_b200_div_by_x_minus_z_dev", (f, a, 16, b, 1, None)),
                  ("sppark_b200_evaluate_dev", (f, b, a, 2, a, 16, None)),
                  ("sppark_b200_batch_inverse_dev", (f, b, a, 16, None))]
    for f in (0, 1):
        calls += [("sppark_b200_ntt_matrix_dev", (f, a, 3, 2, 0, 0, 0, None)),
                  ("sppark_b200_lde_matrix_dev", (f, b, a, 3, 1, 2, None)),
                  ("sppark_b200_ntt_matrix", (f, 0, a, 3, 2, 0, 0, 0)),
                  ("sppark_b200_selftest_word_field", (f, 1, 16, b, a, a))]
    calls.append(("compute_ntt", (0, a, 3, 0, 0, 0)))
    return calls


def test_refusals_after_the_device_lookup(lib):
    if not _no_gpu():
        pytest.skip("a GPU is present; these calls fail only where there is no device")
    u = Bufs()
    for name, args in _after_device_calls(u):
        code, _ = _call(lib, name, *args)
        assert code == NODEV, (name, args, code)
    assert u.unchanged()
