"""cape_b200: H100-native (sm_90a) implementation of CAPE's Chebyshev graph-conv encoder/decoder +
mesh-patch discriminator hot path.  Compute lives in libcape_b200.so (hand-written CUDA, C ABI in
include/cape_b200.h); this package is the host side mirroring the reference's Python API."""
__version__ = "0.1.0"
