"""sppark_b200: H100-native MSM + NTT primitives behind sppark's C ABI.

The product is sppark_b200/libsppark_b200.so (CUDA, sm_90a) and include/sppark_b200.h;
these Python modules are the host-side mirror of the reference's Rust crates, used by the
tests and bench.py.
"""
from . import _lib  # noqa: F401
