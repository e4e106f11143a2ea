"""ctypes loader of libsppark_b200.so.  There is no CPU fallback: if the CUDA library is
missing or the machine has no H100-class (sm_90) device, calls fail loudly."""
import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("SPPARK_B200_LIB") or os.path.join(HERE, "libsppark_b200.so")   # override: experiments only


class RustError(C.Structure):
    """sppark::Error / RustError (rust/src/lib.rs:9-13, util/rusterror.h:18-36)."""
    _fields_ = [("code", C.c_int), ("message", C.c_void_p)]


class GpuPtr(C.Structure):
    """sppark::Gpu_Ptr<T> (rust/src/lib.rs:62-97): one pointer-sized handle."""
    _fields_ = [("inner", C.c_void_p)]


class SpparkError(RuntimeError):
    def __init__(self, code, message):
        super().__init__(f"sppark_b200 error {code}: {message}")
        self.code = code


_lib = None

_SIGS = {
    "mult_pippenger": [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p],
    "mult_pippenger_inf": [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t],
    "mult_pippenger_fp2_inf": [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t],
    "compute_ntt": [C.c_size_t, C.c_void_p, C.c_uint32, C.c_int, C.c_int, C.c_int],
    "sppark_b200_ntt": [C.c_int, C.c_size_t, C.c_void_p, C.c_uint32, C.c_int, C.c_int, C.c_int],
    "sppark_b200_ntt_dev": [C.c_int, C.c_void_p, C.c_uint32, C.c_int, C.c_int, C.c_int, C.c_void_p],
    "sppark_b200_lde": [C.c_int, C.c_size_t, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p],
    "sppark_b200_ntt_slab_pass": [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32,
                                  C.c_int, C.c_void_p],
    "sppark_b200_ntt_slab_pass_p2p": [C.c_int, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32,
                                      C.c_int, C.c_void_p],
    "sppark_b200_peer_alloc": [C.c_size_t, C.POINTER(C.c_void_p), C.c_void_p],
    "sppark_b200_peer_open": [C.c_void_p, C.POINTER(C.c_void_p)],
    "sppark_b200_peer_close": [C.c_void_p],
    "sppark_b200_peer_free": [C.c_void_p],
    "sppark_b200_msm": [C.c_int, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t],
    "sppark_b200_msm_ex": [C.c_int, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_int],
    "sppark_b200_msm_ctx_create": [C.c_int, C.c_void_p, C.c_size_t, C.c_size_t, C.POINTER(C.c_void_p)],
    "sppark_b200_msm_ctx_invoke": [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_int],
    "sppark_b200_msm_dev": [C.c_int, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p],
    "sppark_b200_generate_points_dev": [C.c_int, C.c_void_p, C.c_size_t, C.c_void_p],
    "sppark_b200_msm_combine": [C.c_int, C.c_void_p, C.c_void_p, C.c_size_t],
    "sppark_b200_selftest_field": [C.c_int, C.c_int, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p],
    "sppark_b200_lde_powers_dev": [C.c_int, C.c_void_p, C.c_uint32, C.c_void_p],
    "sppark_b200_lde_expand_dev": [C.c_int, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p],
    "sppark_b200_msm_sharded": [C.c_int, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_int, C.c_void_p, C.c_size_t],
    "sppark_b200_ntt_sharded": [C.c_int, C.c_void_p, C.c_uint32, C.c_int, C.c_void_p, C.c_size_t],
    "sppark_b200_selftest_word_field": [C.c_int, C.c_int, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p],
    "sppark_b200_prefix_op_dev": [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p],
    "sppark_b200_div_by_x_minus_z_dev": [C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_int, C.c_void_p],
    "sppark_b200_evaluate_dev": [C.c_int, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p],
    "sppark_b200_batch_inverse_dev": [C.c_int, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p],
}

# every symbol include/sppark_b200.h declares (tests check the .so exports all of them)
EXPORTS = list(_SIGS) + ["cuda_available", "drop_error_message", "sppark_b200_sm_count", "sppark_b200_ngpus",
                         "sppark_b200_version", "sppark_b200_launch_count",
                         "sppark_b200_profile_enable", "sppark_b200_profile_read",
                         "drop_gpu_ptr_t", "clone_gpu_ptr_t", "sppark_b200_msm_ctx_free", "sppark_b200_gpu_ptr_alloc",
                         "sppark_b200_gpu_ptr_get", "sppark_b200_gpu_ptr_refs"]


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(f"{LIB_PATH} not built: run `python -m sppark_b200.build` "
                              "(there is no CPU fallback)")
        l = C.CDLL(LIB_PATH)
        for name, args in _SIGS.items():
            fn = getattr(l, name)      # every symbol of include/sppark_b200.h must be exported
            fn.argtypes = args
            fn.restype = RustError
        l.cuda_available.restype = C.c_int
        l.drop_error_message.argtypes = [C.c_void_p]
        l.sppark_b200_sm_count.argtypes = [C.c_int]
        l.sppark_b200_version.restype = C.c_char_p
        l.sppark_b200_launch_count.restype = C.c_uint64
        l.sppark_b200_msm_ctx_free.argtypes = [C.c_void_p]
        l.sppark_b200_msm_ctx_free.restype = None
        l.drop_gpu_ptr_t.argtypes = [C.POINTER(GpuPtr)]
        l.clone_gpu_ptr_t.argtypes = [C.POINTER(GpuPtr)]
        l.clone_gpu_ptr_t.restype = GpuPtr
        l.sppark_b200_gpu_ptr_alloc.argtypes = [C.c_size_t]
        l.sppark_b200_gpu_ptr_alloc.restype = GpuPtr
        l.sppark_b200_gpu_ptr_get.argtypes = [C.POINTER(GpuPtr)]
        l.sppark_b200_gpu_ptr_get.restype = C.c_void_p
        l.sppark_b200_gpu_ptr_refs.argtypes = [C.POINTER(GpuPtr)]
        l.sppark_b200_gpu_ptr_refs.restype = C.c_size_t
        l.sppark_b200_profile_enable.argtypes = [C.c_int]
        l.sppark_b200_profile_read.argtypes = [C.POINTER(C.c_char_p), C.POINTER(C.c_float), C.c_int]
        l.sppark_b200_profile_read.restype = C.c_int
        _lib = l
    return _lib


def check(err):
    """Turn a by-value RustError into an exception, freeing the message like Rust's
    `impl From<Error> for String` does (rust/src/lib.rs:15-22)."""
    if err.code != 0:
        msg = C.cast(err.message, C.c_char_p).value.decode() if err.message else ""
        if err.message:
            lib().drop_error_message(err.message)
        raise SpparkError(err.code, msg)


def launch_count():
    return int(lib().sppark_b200_launch_count())


def profile_enable(on=True):
    lib().sppark_b200_profile_enable(int(on))


def profile_read():
    """[(phase, ms)] of the last profiled call (synchronise first)."""
    names = (C.c_char_p * 16)()
    ms = (C.c_float * 16)()
    n = lib().sppark_b200_profile_read(names, ms, 16)
    return [(names[i].decode(), float(ms[i])) for i in range(n)]
