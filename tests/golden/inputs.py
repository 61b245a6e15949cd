"""Seeded inputs of the golden op cases (shared by make_golden.py and the tests; outputs are committed)."""
import hashlib

import numpy as np

# ops_golden.npz keeps every OPS_VSTRIDE-th vertex of each output (the file stays under 1 MB)
OPS_VSTRIDE = 4


def digest(a):
    """SHA-256 of an array's dtype, shape and bytes: what lap_golden.npz stores for a bit-for-bit comparison."""
    a = np.ascontiguousarray(a)
    return hashlib.sha256(("%s%s" % (a.dtype.str, a.shape)).encode() + a.tobytes()).hexdigest()


def golden_inputs():
    rng = np.random.RandomState(123)
    g = {}
    g["c1_x"] = rng.normal(size=(1, 6890, 3)).astype(np.float32)
    g["c1_W"] = np.clip(rng.normal(0, 0.1, size=(18, 64)), -0.2, 0.2).astype(np.float32)
    g["cnp_x"] = rng.normal(size=(2, 6890, 16)).astype(np.float32)
    g["cnp_W"] = np.clip(rng.normal(0, 0.1, size=(32, 32)), -0.2, 0.2).astype(np.float32)
    g["cnp_b"] = rng.normal(0, 0.1, size=(32,)).astype(np.float32)
    g["up_x"] = rng.normal(size=(2, 3445, 8)).astype(np.float32)
    return g
