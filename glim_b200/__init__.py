"""glim_b200: H100-native (sm_90a) VGICP scan-matching hot path of koide3/glim behind the gtsam_points class
surface GLIM uses.  The compute lives in libglim_b200.so (CUDA, C-ABI: include/glim_b200.h); this package is the
thin host mirror used by tests and the bench.  No CPU fallback: importing is cheap, calling without the built
library or without an H100 raises."""
from . import capi  # noqa: F401

__all__ = ["capi"]
