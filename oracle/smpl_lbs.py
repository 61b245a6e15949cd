"""Float64 numpy transcription of the SMPL forward pass that demo_full poses clothed meshes with (demos.py:249-331 of the
reference: smplx's `lbs` with zero betas and v_template replaced by the clothed mesh).  Test infrastructure only."""
import numpy as np


def rodrigues(r):
    """[..., 3] axis-angle -> [..., 3, 3] rotation matrices, as smplx.lbs.batch_rodrigues (angle of r + 1e-8)."""
    r = np.asarray(r, np.float64)
    angle = np.linalg.norm(r + 1e-8, axis=-1, keepdims=True)
    d = r / angle
    x, y, z = d[..., 0], d[..., 1], d[..., 2]
    zero = np.zeros_like(x)
    K = np.stack([zero, -z, y, z, zero, -x, -y, x, zero], -1).reshape(r.shape[:-1] + (3, 3))
    s, c = np.sin(angle)[..., None], np.cos(angle)[..., None]
    return np.eye(3) + s * K + (1 - c) * (K @ K)


def relative_transforms(J, R, parents):
    """Joints [24, 3], rotations [24, 3, 3] -> (global transforms G [24, 4, 4], A = G - G . [J, 0])."""
    n = len(parents)
    G = np.zeros((n, 4, 4))
    for j in range(n):
        T = np.eye(4)
        T[:3, :3] = R[j]
        T[:3, 3] = J[j] - (J[parents[j]] if parents[j] >= 0 else 0.0)
        G[j] = T if parents[j] < 0 else G[parents[j]] @ T
    A = G.copy()
    A[:, :3, 3] -= np.einsum("jab,jb->ja", G[:, :3, :3], J)
    return G, A


def lbs(v_template, pose, J_regressor, posedirs, weights, parents):
    """One mesh: v_template [V, 3] (the clothed mesh), pose [72], J_regressor [24, V] (dense or scipy), posedirs
    [V, 3, 207] (the pickle's layout), weights [V, 24], parents [24] (root -1) -> posed vertices [V, 3]."""
    v = np.asarray(v_template, np.float64)
    J = np.asarray(J_regressor @ v, np.float64)
    R = rodrigues(np.asarray(pose, np.float64).reshape(-1, 3))
    pose_feature = (R[1:] - np.eye(3)).reshape(-1)
    v_posed = v + np.einsum("vcp,p->vc", np.asarray(posedirs, np.float64), pose_feature)
    _, A = relative_transforms(J, R, parents)
    T = np.einsum("vj,jab->vab", np.asarray(weights, np.float64), A)
    return np.einsum("vab,vb->va", T[:, :3, :3], v_posed) + T[:, :3, 3]


def lbs_batch(verts, poses, model):
    """[N, V, 3] meshes, [N, 72] poses, model = dict of the pickle's arrays (J_regressor, posedirs, weights, parents)."""
    return np.stack([lbs(v, p, model["J_regressor"], model["posedirs"], model["weights"], model["parents"])
                     for v, p in zip(verts, poses)])
