"""bundletrack_b200 — H100-native (sm_90a) pose-graph optimizer + feature matcher that drops in behind
BundleTrack's C++ surface.  The product is lib/libbundletrack_b200.so (hand-written CUDA behind a C-ABI, see
include/bundletrack_b200.h); this package is the thin Python host used by tests and bench.py."""
from . import _lib  # noqa: F401
from .config import solver_params  # noqa: F401
