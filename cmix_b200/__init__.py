"""cmix_b200 — H100-native per-bit context-mixing predictor behind cmix's Predictor surface.

The product is the C-ABI shared library built from cmix_b200/csrc (see include/cmixb200.h);
this package is the thin Python binding used by tests/ and bench.py. It never falls back to
a CPU implementation: importing it without the built library raises.
"""
import os as _os

# Many independent files run on 3 CUDA streams per launch group; the default of 8 hardware work queues
# would alias them and serialise independent groups. Must be set before the CUDA context exists.
_os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")

from .capi import Predictor, load_library, build_library, N_EXT, LIB_PATH  # noqa: F401
