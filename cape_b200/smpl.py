"""SMPL body model for demo_full: posing of clothed meshes on the GPU (what the reference gets from `smplx` on CPU
torch, demos.py:22-24,249-331), and the pose-vector / rotation-matrix conversions of lib/utils.py:80-111 without cv2.

The body model is the user's own licensed file `<smpl_model_folder>/smpl/SMPL_<GENDER>.pkl`, the official SMPL pickle
with the chumpy objects removed (smplx reads the same file).  Posing follows smplx.lbs with zero shape parameters and
the template replaced by the mesh to pose -- the joints are regressed from that mesh -- as the reference does.
"""
import os
import pickle

import numpy as np
import scipy.sparse as sp
import torch

N_JOINTS = 24


def model_path(smpl_model_folder, gender):
    """The file smplx.create(model_type='smpl', model_path=folder, gender=gender) reads."""
    return os.path.join(smpl_model_folder, "smpl", "SMPL_%s.pkl" % gender.upper())


def load_model(path):
    """The arrays of an SMPL pickle: v_template [V, 3], f [F, 3], posedirs [V, 3, 207], weights [V, 24], J_regressor
    (scipy CSR [24, V]) and parents [24] (kintree_table[0] with the root's entry set to -1, as smplx does)."""
    if not os.path.exists(path):
        raise FileNotFoundError("SMPL model not found: %s (the official SMPL pickle; README.md, 'Test and demo modes')"
                                % path)
    with open(path, "rb") as f:
        data = pickle.load(f, encoding="latin1")
    out = {"v_template": np.asarray(data["v_template"], np.float64), "f": np.asarray(data["f"], np.int64),
           "posedirs": np.asarray(data["posedirs"], np.float64), "weights": np.asarray(data["weights"], np.float64),
           "J_regressor": sp.csr_matrix(data["J_regressor"], dtype=np.float64)}
    parents = np.asarray(data["kintree_table"])[0].astype(np.int64)
    parents[0] = -1
    out["parents"] = parents
    V = out["v_template"].shape[0]
    if out["weights"].shape != (V, N_JOINTS) or out["J_regressor"].shape != (N_JOINTS, V):
        raise ValueError("%s: weights %s / J_regressor %s do not fit %d vertices and %d joints"
                         % (path, out["weights"].shape, out["J_regressor"].shape, V, N_JOINTS))
    if out["posedirs"].shape != (V, 3, 9 * (N_JOINTS - 1)):
        raise ValueError("%s: posedirs has shape %s, expected %s" % (path, out["posedirs"].shape, (V, 3, 207)))
    return out


class SMPL(object):
    """Device-resident SMPL model (cape_smpl): `pose(verts [N, V, 3], pose72 [N, 72]) -> posed verts`, numpy in/out.
    `model`: a dict as load_model returns, or the path of a pickle."""

    def __init__(self, model, device=0):
        from .engine import SmplPoser
        if isinstance(model, str):
            model = load_model(model)
        self.model = model
        self.faces = model["f"]
        V = model["v_template"].shape[0]
        J = sp.csr_matrix(model["J_regressor"])
        J.sort_indices()
        posedirs = np.asarray(model["posedirs"]).reshape(V * 3, -1).T          # [207, V*3], as smplx stores it
        self.poser = SmplPoser(J.indptr, J.indices, J.data, posedirs, model["weights"], model["parents"], device)

    def pose(self, verts, pose):
        verts = np.asarray(verts)
        pose = np.asarray(pose)
        if verts.ndim != 3 or pose.shape != (verts.shape[0], 72):
            raise ValueError("pose() takes verts [N, V, 3] and pose [N, 72], got %s and %s" % (verts.shape, pose.shape))
        dev = self.poser.device
        v = torch.from_numpy(np.ascontiguousarray(verts, np.float32)).to(dev)
        p = torch.from_numpy(np.ascontiguousarray(pose, np.float32)).to(dev)
        out = torch.empty_like(v)
        self.poser.pose(v, p, out)
        return out.cpu().numpy()


# ---------------------------------------------------------------------------------------------------------------------
# lib/utils.py:80-111 (cv2.Rodrigues) in numpy
# ---------------------------------------------------------------------------------------------------------------------
def _vec2mat(r):
    theta = np.linalg.norm(r)
    if theta < np.finfo(np.float64).eps:
        return np.eye(3)
    c, s = np.cos(theta), np.sin(theta)
    x, y, z = r / theta
    rrt = np.outer([x, y, z], [x, y, z])
    r_x = np.array([[0, -z, y], [z, 0, -x], [-y, x, 0]])
    return c * np.eye(3) + (1 - c) * rrt + s * r_x


def _mat2vec(R):
    # cv2.Rodrigues: orthonormalise first (nearest rotation through the SVD), then read the angle and axis; the axis of
    # a half turn comes from the diagonal
    U, _, Vt = np.linalg.svd(R)
    R = U @ Vt
    r = np.array([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]])
    s = np.sqrt((r @ r) * 0.25)
    c = np.clip((R[0, 0] + R[1, 1] + R[2, 2] - 1) * 0.5, -1.0, 1.0)
    theta = np.arccos(c)
    if s >= 1e-5:
        return r * (theta / (2 * s))
    if c > 0:
        return np.zeros(3)
    r = np.array([np.sqrt(max((R[0, 0] + 1) * 0.5, 0.0)),
                  np.sqrt(max((R[1, 1] + 1) * 0.5, 0.0)) * (-1.0 if R[0, 1] < 0 else 1.0),
                  np.sqrt(max((R[2, 2] + 1) * 0.5, 0.0)) * (-1.0 if R[0, 2] < 0 else 1.0)])
    if abs(r[0]) < abs(r[1]) and abs(r[0]) < abs(r[2]) and (R[1, 2] > 0) != (r[1] * r[2] > 0):
        r[2] = -r[2]
    return r * (theta / np.linalg.norm(r))


def pose2rot(pose):
    """[n, 72] axis-angle pose vectors -> [n, 216] flattened rotation matrices (lib/utils.py:80-94)."""
    pose = np.asarray(pose)
    n = pose.shape[0]
    out = np.array([np.concatenate([_vec2mat(v).ravel() for v in p.reshape(-1, 3).astype(np.float64)]) for p in pose])
    return out.reshape(n, -1).astype(pose.dtype if pose.dtype.kind == "f" else np.float64)


def rot2pose(rot):
    """[n, 216] flattened rotation matrices -> [n, 72] axis-angle pose vectors (lib/utils.py:96-110)."""
    rot = np.asarray(rot)
    n = rot.shape[0]
    out = np.array([np.concatenate([_mat2vec(m.reshape(3, 3)) for m in r.reshape(-1, 9).astype(np.float64)]) for r in rot])
    return out.reshape(n, -1).astype(rot.dtype if rot.dtype.kind == "f" else np.float64)
