#!/usr/bin/env python
"""Converter: the reference checkout's operator fixtures -> pickle-free .npz fixtures under tests/golden/.

The reference ships its fixed mesh hierarchy as pickled scipy CSC matrices
(<CAPE checkout>/data/transform_matrices/{for_demo,ds2}/{A,D,U}.npy, loaded at lib/load_data.py:7-32 with
encoding='latin1').  Those files are the fixed SMPL mesh hierarchy every model of CAPE runs on, so the
repository keeps this converted copy as test data (tests/golden/smpl_topology_{for_demo,ds2,assets}.npz, split to keep
each file small); the package loads its hierarchy from there.  Licence: the files are derived from data the reference
distributes under its own licence (its LICENSE file: no redistribution; the template mesh and edge table are SMPL data
under the SMPL licence).  They are kept here as test fixtures of that data; whoever redistributes this repository must
have the right to redistribute them.
It holds the operators as plain CSR arrays
(indptr/indices/data/shape), the SMPL edge table (data/edges_smpl.npy, used by lib/losses.py:9-25; = upper triangle
of A[0], checked against the reference file), the per-vertex normalisation statistics
(data/demo_data/trainset_stats.npz, demos.py:155), the clothing-vertex index list, the template mesh and the demo
poses (demos.py:349-357).

    python -m cape_b200.pack_topology --reference /path/to/CAPE        (default: $CAPE_REFERENCE)
"""
import argparse
import os
import sys
import numpy as np
import scipy.sparse as sp

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
PARTS = ("for_demo", "ds2", "assets")     # one file per hierarchy; the edge table, statistics and demo assets


def default_reference():
    """The reference checkout to read the fixtures from: $CAPE_REFERENCE; None if unset or absent."""
    cand = os.environ.get("CAPE_REFERENCE")
    if cand and os.path.isdir(os.path.join(cand, "data", "transform_matrices")):
        return cand
    return None


def pack(REF, OUT=OUT):
    def _load(kind, name):
        path = os.path.join(REF, "data", "transform_matrices", kind, name + ".npy")
        return list(np.load(path, encoding="latin1", allow_pickle=True))

    out = {}
    for kind in ("for_demo", "ds2"):
        for name in ("A", "D", "U"):
            mats = _load(kind, name)
            out[f"{kind}.{name}.count"] = np.int64(len(mats))
            for i, m in enumerate(mats):
                m = sp.csr_matrix(m)
                m.sort_indices()
                key = f"{kind}.{name}.{i}"
                out[key + ".indptr"] = m.indptr.astype(np.int32)
                out[key + ".indices"] = m.indices.astype(np.int32)
                out[key + ".data"] = m.data  # dtype kept (for_demo fp32, ds2 fp64)
                out[key + ".shape"] = np.asarray(m.shape, np.int64)
    a0 = sp.coo_matrix(_load("for_demo", "A")[0])
    keep = a0.row < a0.col
    edges = np.stack([a0.row[keep], a0.col[keep]], 1).astype(np.int32)
    edges = edges[np.lexsort((edges[:, 1], edges[:, 0]))]
    ref_edges = np.load(os.path.join(REF, "data", "edges_smpl.npy"))
    assert set(map(tuple, edges.tolist())) == set(map(tuple, np.sort(ref_edges, 1).tolist()))
    out["edges"] = edges
    st = np.load(os.path.join(REF, "data", "demo_data", "trainset_stats.npz"))
    out["stats.mean"] = st["mean"].astype(np.float32)
    out["stats.std"] = st["std"].astype(np.float32)
    out["clothing_verts_idx"] = np.load(os.path.join(REF, "data", "clothing_verts_idx.npy")).astype(np.int32)
    # demo assets (demos.py:351-357): template mesh (minimal body shape + faces) and the demo poses
    v, f = [], []
    for ln in open(os.path.join(REF, "data", "template_mesh.obj")):
        t = ln.split()
        if t and t[0] == "v":
            v.append([float(x) for x in t[1:4]])
        elif t and t[0] == "f":
            f.append([int(x.split("/")[0]) - 1 for x in t[1:4]])
    out["template.v"], out["template.f"] = np.asarray(v, np.float64), np.asarray(f, np.int32)
    dp = np.load(os.path.join(REF, "data", "demo_data", "demo_pose_params.npz"))
    out["demo.rot"], out["demo.pose"] = dp["rot"], dp["pose"]
    os.makedirs(OUT, exist_ok=True)
    for name in PARTS:
        keys = [k for k in out if k.split(".")[0] == name or (name == "assets" and k.split(".")[0] not in PARTS)]
        np.savez_compressed(os.path.join(OUT, "smpl_topology_%s.npz" % name), **{k: out[k] for k in keys})
    return OUT


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--reference", default=default_reference(), help="checkout of qianlim/CAPE")
    ap.add_argument("--out", default=OUT, help="directory of the two .npz files")
    a = ap.parse_args(argv)
    if not a.reference:
        ap.error("no reference checkout found: pass --reference or set CAPE_REFERENCE")
    out = pack(a.reference, a.out)
    print("wrote smpl_topology_{%s}.npz to %s" % (",".join(PARTS), os.path.abspath(out)))


if __name__ == "__main__":
    sys.exit(main())
