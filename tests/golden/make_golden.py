#!/usr/bin/env python
"""Generate the committed golden vectors.  Needs a reference checkout ($CAPE_REFERENCE).

What it pins (the reference ships no tests of its own, SURVEY.md section 4):
  1. rescaled Laplacians produced by the REFERENCE's own host code (lib/mesh_sampling.py laplacian +
     rescale_L, imported from the reference checkout) for every level of both hierarchies -> lap_golden.npz.
     cape_b200.topology and oracle/ must reproduce them bit for bit.
  2. known answers of the op bodies from the literal numpy transcription (oracle/np_ops.py), cross-checked
     here against the independent float64 dense-polynomial formulation -> ops_golden.npz:
       C1: single Chebyshev K=6 layer on a [1,6890,3] input (BASELINE.json configs[0]),
       a K=2 64->32 conv + bias/leaky-ReLU + pool on level 1, and an unpool.
"""
import os
import sys

import numpy as np
import scipy.sparse as sp

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.abspath(os.path.join(HERE, "..", ".."))
REF = os.environ.get("CAPE_REFERENCE", "")
sys.path.insert(0, ROOT)
sys.path.insert(0, REF)
sys.path.insert(0, HERE)

from lib import mesh_sampling as ref_ms  # noqa: E402  (the reference's own module)
from inputs import OPS_VSTRIDE, digest, golden_inputs  # noqa: E402
from oracle import np_ops  # noqa: E402


def load(kind, name):
    return list(np.load(os.path.join(REF, "data", "transform_matrices", kind, name + ".npy"), encoding="latin1",
                        allow_pickle=True))


def main():
    out = {}
    for kind in ("for_demo", "ds2"):
        A = [a.astype("float32") for a in load(kind, "A")]
        for i, a in enumerate(A):
            L = ref_ms.laplacian(a, normalized=True)
            Lt = sp.csr_matrix(ref_ms.rescale_L(sp.csr_matrix(L), lmax=2))
            Lt.sort_indices()
            L = sp.csr_matrix(L)
            L.sort_indices()
            for tag, m in (("L", L), ("Lt", Lt)):
                k = "%s.%s.%d" % (kind, tag, i)
                for part in ("indptr", "indices", "data"):
                    out[k + "." + part] = np.array(digest(getattr(m, part)))
    np.savez_compressed(os.path.join(HERE, "lap_golden.npz"), **out)

    g = golden_inputs()
    A = [a.astype("float32") for a in load("for_demo", "A")]
    D = [d.astype("float32") for d in load("for_demo", "D")]
    U = [u.astype("float32") for u in load("for_demo", "U")]
    L0 = ref_ms.laplacian(A[0], normalized=True)
    L1 = ref_ms.laplacian(A[1], normalized=True)
    ops = {}
    # C1: K=6, [1,6890,3] -> 64 (BASELINE.json configs[0])
    y = np_ops.chebyshev5_np(g["c1_x"], L0, g["c1_W"], 6)
    y64 = np_ops.chebyshev_dense_f64(g["c1_x"], L0, g["c1_W"], 6)
    err = np.abs(y - y64).max() / np.abs(y64).max()
    assert err < 1e-5, err
    ops["c1_y"] = y.astype(np.float32)[:, ::OPS_VSTRIDE]
    # K=2 conv 16->32 + bias + leaky + pool D[1] (6890 -> 3445), batch 2
    y2 = np_ops.poolwT_np(np_ops.b1leakyrelu_np(np_ops.chebyshev5_np(g["cnp_x"], L1, g["cnp_W"], 2), g["cnp_b"]), D[1])
    ops["cnp_y"] = y2.astype(np.float32)[:, ::OPS_VSTRIDE]
    # unpool U[1] (3445 -> 6890)
    ops["up_y"] = np_ops.poolwT_np(g["up_x"], U[1]).astype(np.float32)[:, ::OPS_VSTRIDE]
    np.savez_compressed(os.path.join(HERE, "ops_golden.npz"), **ops)
    print("golden vectors written; C1 literal-vs-f64 rel err %.2e" % err)


if __name__ == "__main__":
    main()
