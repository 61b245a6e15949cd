"""The test / demo modes without a GPU: the numpy Rodrigues conversions against cv2, the float64 SMPL oracle against
independent facts, the SMPL pickle loader, and our demo_full against what the reference's demo_full did with the same
stand-ins (tests/golden/make_demo_full_golden.py -> demo_full_golden.npz)."""
import os
import pickle

import numpy as np
import pytest
import scipy.sparse as sp

import make_demo_full_golden as DG
from cape_b200 import demos, smpl
from cape_b200 import topology as T
from oracle import smpl_lbs

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "demo_full_golden.npz")
# SMPL's kinematic tree (kintree_table[0]; the pickle's root entry is not a valid index)
SMPL_PARENTS = [-1, 0, 0, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 9, 9, 12, 13, 14, 16, 17, 18, 19, 20, 21]


@pytest.fixture(scope="module")
def golden():
    with np.load(GOLDEN) as z:
        return {k: z[k] for k in z.files}


def synthetic_smpl(seed=0, V=None):
    """An SMPL model with the real template and tree: weight rows summing to 1 with at most 4 non-zeros, J_regressor
    rows summing to 1 (sparse), posedirs of magnitude ~1e-2."""
    rng = np.random.RandomState(seed)
    v, f = T.template_mesh()
    V = V or len(v)
    v = v[:V]
    weights = np.zeros((V, 24))
    for i in range(V):
        js = rng.choice(24, size=rng.randint(1, 5), replace=False)
        w = rng.uniform(0.1, 1.0, size=len(js))
        weights[i, js] = w / w.sum()
    jreg = np.zeros((24, V))
    for j in range(24):
        cols = rng.choice(V, size=12, replace=False)
        w = rng.uniform(0.1, 1.0, size=12)
        jreg[j, cols] = w / w.sum()
    return {"v_template": v, "f": f[(f < V).all(1)], "posedirs": rng.normal(size=(V, 3, 207)) * 1e-2,
            "shapedirs": np.zeros((V, 3, 10)), "weights": weights, "J_regressor": sp.csc_matrix(jreg),
            "kintree_table": np.stack([np.array([4294967295] + SMPL_PARENTS[1:], np.int64), np.arange(24)])}


def write_pickle(folder, gender, model):
    path = smpl.model_path(str(folder), gender)
    os.makedirs(os.path.dirname(path), exist_ok=True)
    with open(path, "wb") as f:
        pickle.dump(model, f, protocol=2)
    return path


# ---- pose2rot / rot2pose ---------------------------------------------------------------------------------------------
def test_rodrigues_conversions_match_cv2(golden):
    rot, pose = T.demo_pose_params()
    assert np.abs(smpl.rot2pose(rot) - golden["utils/rot2pose_demo"]).max() < 1e-6
    assert np.abs(smpl.pose2rot(pose) - golden["utils/pose2rot_demo"]).max() < 1e-6
    assert np.abs(smpl.pose2rot(golden["utils/near_pose"]) - golden["utils/pose2rot_near"]).max() < 1e-6
    assert np.abs(smpl.rot2pose(golden["utils/near_rot"]) - golden["utils/rot2pose_near"]).max() < 1e-6
    assert np.abs(smpl.pose2rot(pose) - rot).max() < 1e-6              # the shipped demo.rot are pose2rot(demo.pose)


# ---- the float64 oracle --------------------------------------------------------------------------------------------
def _oracle_model(m):
    return {"J_regressor": sp.csr_matrix(m["J_regressor"]), "posedirs": m["posedirs"], "weights": m["weights"],
            "parents": np.array(SMPL_PARENTS)}


def test_oracle_zero_pose_returns_the_template():
    m = synthetic_smpl(1)
    out = smpl_lbs.lbs_batch(m["v_template"][None], np.zeros((1, 72)), _oracle_model(m))[0]
    assert np.abs(out - m["v_template"]).max() < 1e-12


def test_oracle_vertex_bound_to_one_joint_moves_rigidly():
    m = synthetic_smpl(2)
    m["weights"][0] = np.eye(24)[18]
    mm = _oracle_model(m)
    pose = np.random.RandomState(0).normal(size=72) * 0.5
    v = m["v_template"]
    J = mm["J_regressor"] @ v
    R = smpl_lbs.rodrigues(pose.reshape(-1, 3))
    G, _ = smpl_lbs.relative_transforms(J, R, SMPL_PARENTS)
    pf = (R[1:] - np.eye(3)).reshape(-1)
    v_posed = v[0] + m["posedirs"][0] @ pf
    want = G[18, :3, :3] @ (v_posed - J[18]) + G[18, :3, 3]        # rigid motion of joint 18's frame
    got = smpl_lbs.lbs(v, pose, mm["J_regressor"], m["posedirs"], m["weights"], SMPL_PARENTS)[0]
    assert np.abs(got - want).max() < 1e-12


def test_oracle_rodrigues_agrees_with_scipy():
    from scipy.spatial.transform import Rotation
    r = np.random.RandomState(4).normal(size=(200, 3))
    r *= (np.random.RandomState(5).uniform(0, np.pi, size=200) / np.linalg.norm(r, axis=1))[:, None]
    assert np.abs(smpl_lbs.rodrigues(r) - Rotation.from_rotvec(r).as_matrix()).max() < 1e-7
    assert np.array_equal(smpl_lbs.rodrigues(np.zeros((1, 3)))[0], np.eye(3))


# ---- the SMPL pickle loader ----------------------------------------------------------------------------------------
def test_smpl_loader_reads_the_official_layout(tmp_path):
    m = synthetic_smpl(3, V=300)
    path = write_pickle(tmp_path, "female", m)
    assert path == os.path.join(str(tmp_path), "smpl", "SMPL_FEMALE.pkl")
    got = smpl.load_model(path)
    assert list(got["parents"]) == SMPL_PARENTS
    assert sp.issparse(got["J_regressor"]) and np.array_equal(got["J_regressor"].toarray(), m["J_regressor"].toarray())
    for k in ("v_template", "posedirs", "weights"):
        assert np.array_equal(got[k], m[k])
    assert np.array_equal(got["f"], m["f"])


def test_smpl_loader_names_a_missing_file(tmp_path):
    path = smpl.model_path(str(tmp_path), "male")
    with pytest.raises(FileNotFoundError, match=path.replace("\\", "\\\\")):
        smpl.load_model(path)


# ---- demo_full against the reference's ---------------------------------------------------------------------------
class StandinBody(object):
    """The golden generator's stand-in body model behind our demo_full's body_model interface, recording the calls."""

    def __init__(self):
        self.faces = T.template_mesh()[1]
        self.calls = []

    def pose(self, verts, poses):
        out = []
        for v, p in zip(verts, poses):
            v32, p32 = np.asarray(v, np.float32), np.asarray(p, np.float32)
            self.calls.append((v32[::DG.VSTRIDE], p32[:3], p32[3:]))
            out.append(DG.standin_pose(v32, p32[:3], p32[3:]))
        return np.stack(out)


def test_demo_full_equals_the_references(golden, tmp_path):
    model, body = DG.DemoModel(), StandinBody()
    res = str(tmp_path / "results" / "run")
    d = demos.demo_full(model, "run", "male", "dset", "unused", "unused", n_sample=DG.N_SAMPLE, save_obj=True,
                        random_seed=123, vis=False, body_model=body, results_dir=res)
    d.run()
    d.n_sample = DG.TEST_N_SAMPLE
    out = d.test_model(DG.body_data())
    # decode calls: the same latent draws and condition embeddings (rot[0] conditions the clothing-type demo)
    assert len(model.decode_calls) == len(golden["decode/z"]) == 6 + 4
    for (z, c, c2), gz, gc, gc2 in zip(model.decode_calls, golden["decode/z"], golden["decode/cond"], golden["decode/cond2"]):
        assert np.abs(z - gz).max() < 1e-6 and np.abs(c - gc).max() < 1e-6 and np.abs(c2 - gc2).max() < 1e-6
    # the body model sees what the reference's smplx model was given for every mesh it wrote (pose[2] for the clothing
    # types, the exemplar stride of the test set); the reference's extra posing of the bare template is not repeated
    written = golden["body/written"]
    assert len(body.calls) == int(written.sum())
    for (v, go, bp), gv, ggo, gbp in zip(body.calls, golden["body/v"][written], golden["body/global_orient"][written],
                                         golden["body/body_pose"][written]):
        assert np.abs(v - gv).max() < 1e-5
        assert np.abs(go - ggo).max() < 1e-6 and np.abs(bp - gbp).max() < 1e-6
    # OBJ files: same names, same order, same vertices
    paths = sorted(os.path.relpath(os.path.join(r, f), res) for r, _, fs in os.walk(res) for f in fs if f.endswith(".obj"))
    assert paths == sorted(golden["obj/paths"])
    assert len(golden["obj/paths"]) == 6 * DG.N_SAMPLE + 4 * DG.N_SAMPLE + 4            # stride 3 over 11: 4 > n_sample
    for p, gv in zip(golden["obj/paths"], golden["obj/verts"]):
        v, f = demos.read_obj(os.path.join(res, str(p)))
        assert np.array_equal(f, body.faces)
        assert np.abs(v[::DG.VSTRIDE] - gv).max() < 1e-5, p
    # the order of the writes: the posing calls are in the reference's order
    assert [c[2][:3].tolist() for c in body.calls] == [g[:3].tolist() for g in golden["body/body_pose"][written]]
    # the test-result string and both result files
    assert out["string"] == str(golden["test/string"])
    assert open(os.path.join(res, "test_results_dset.txt")).read() == str(golden["test/string"])
    assert open(os.path.join(res, "..", "all_test_results_dset.txt")).read() == str(golden["test/all_file"])
    assert len(out["posed"]) == 4
