"""bin_b200 -- Hopper-native (H100, sm_90a) implementation of the BIN deblur+interpolation hot path.

Python here is host-side plumbing only (module mirror, weight packing cache, window sharding);
all arithmetic runs in hand-written CUDA kernels inside libbin_b200.so (see include/bin_b200.h).
"""
from ._lib import BinB200Error, lib  # noqa: F401

__version__ = "0.1.0"
