"""gssdf_b200: host-side mirror of the GS-SDF splat / SDF operator surface over libgssdf_b200.so.

The compute lives in hand-written sm_90a CUDA behind the C ABI of include/gssdf_b200.h; this package is
the Python twin of the reference's libtorch wrappers (gsplat_cpp / tcnn_binding). No CPU fallback.
"""
from . import scene  # noqa: F401  (numpy only)
