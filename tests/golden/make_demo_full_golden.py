#!/usr/bin/env python
"""Golden data for the test / demo modes (tests/test_demo_full.py): what the REFERENCE's own `demos.demo_full`
(demos.py:9-336, imported unmodified) does with the stand-ins defined here, written to demo_full_golden.npz:

  * every `decode` call (latent codes and condition embeddings);
  * every call of the body model (the template it was given, every VSTRIDE-th vertex, global orientation and body
    pose) and whether its result was written;
  * every OBJ write, in order: the path relative to the results folder and every VSTRIDE-th vertex;
  * the test-result string of `test_model` and the text of the two result files;
  * `lib/utils.pose2rot` / `rot2pose` (cv2.Rodrigues) on the shipped demo poses and on rotations near 0 and near pi.

smplx, psbody.mesh and trimesh are replaced by stand-ins; the body model's output is a fixed function of its inputs
(`standin_pose`), so the tests can drive our demo_full with the same function.  Runs only where a reference checkout
exists ($CAPE_REFERENCE) and cv2 is installed; the tests read the .npz.

    CAPE_REFERENCE=/path/to/CAPE python tests/golden/make_demo_full_golden.py
"""
import contextlib
import importlib.util
import io
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "demo_full_golden.npz")
VSTRIDE = 29                  # vertices kept of every mesh
N_SAMPLE = 2                  # demo_n_sample of the recorded run
N_TEST = 11                   # test meshes: the exemplar stride int(11 / 3) = 3 gives 4 > n_sample meshes
TEST_N_SAMPLE = 3
NEAR_ANGLES = (0.0, 1e-9, 1e-6, 1e-3, 0.5, np.pi - 1e-3, np.pi - 1e-6, np.pi - 1e-9, np.pi)

sys.path.insert(0, HERE)
import make_host_golden as H  # noqa: E402


# ---------------------------------------------------------------------------------------------------------------
# stand-ins shared by the reference side (here) and our side (the tests)
# ---------------------------------------------------------------------------------------------------------------
def standin_pose(v_template, global_orient, body_pose):
    """The stand-in body model's output: a fixed function of all three inputs, computed from their fp32 values (the
    reference hands them to smplx's fp32 buffers)."""
    v, go, bp = (np.asarray(a, np.float32).astype(np.float64).reshape(s) for a, s in
                 ((v_template, (-1, 3)), (global_orient, (3,)), (body_pose, (69,))))
    s = 1.0 + 0.1 * np.tanh(bp @ np.cos(np.arange(69) * 0.7))
    return (v * s + 0.1 * np.tanh(go) + 0.01 * bp[:3]).astype(np.float32)


class DemoModel(H.FakeModel):
    """demo_simple's stand-in CAPE plus `predict`, recording every decode call."""

    def __init__(self):
        self.decode_calls = []

    def decode(self, data, cond=None, cond2=None):
        self.decode_calls.append((np.asarray(data, np.float32), np.asarray(cond, np.float32), np.asarray(cond2, np.float32)))
        return H.FakeModel.decode(self, data, cond, cond2)

    def predict(self, data, cond=None, cond2=None, labels=None, sess=None, phase="train"):
        x = np.asarray(data, np.float64)
        c, c2 = np.asarray(cond, np.float64), np.asarray(cond2, np.float64)
        pred = (np.tanh(x) * 0.9 + (c.sum(1) * 1e-3 - c2 @ np.arange(4.0) * 1e-3)[:, None, None]).astype(np.float32)
        return pred, float(np.abs(x).mean()), float((x ** 2).mean() * 0.1), float(np.abs(x).max())


def body_data():
    """A small stand-in BodyData whose full test poses are 216-dim rotation matrices."""
    from cape_b200.demos import filter_cloth_pose
    from cape_b200.smpl import pose2rot
    rng = np.random.RandomState(7)
    full = pose2rot(rng.normal(size=(N_TEST, 72)) * 0.4)
    return types.SimpleNamespace(
        vertices_test=rng.normal(size=(N_TEST, 6890, 3)).astype(np.float32),
        cond1_test=filter_cloth_pose(full).astype(np.float32),
        cond2_test=np.eye(4, dtype=np.float32)[rng.randint(0, 4, size=N_TEST)],
        cond1_test_full=full,
        mean=rng.normal(size=(6890, 3)) * 0.02, std=np.abs(rng.normal(size=(6890, 3))) * 0.01 + 0.005)


def near_rotations():
    """Axis-angle poses at the angles of NEAR_ANGLES (random axes) and their exact rotation matrices (scipy)."""
    from scipy.spatial.transform import Rotation
    rng = np.random.RandomState(3)
    axes = rng.normal(size=(len(NEAR_ANGLES), 24, 3))
    axes /= np.linalg.norm(axes, axis=-1, keepdims=True)
    pose = (axes * np.asarray(NEAR_ANGLES)[:, None, None]).reshape(len(NEAR_ANGLES), 72)
    rot = Rotation.from_rotvec(pose.reshape(-1, 3)).as_matrix().reshape(len(NEAR_ANGLES), 216)
    return pose, rot


# ---------------------------------------------------------------------------------------------------------------
# the reference side
# ---------------------------------------------------------------------------------------------------------------
def ref_demo_full(ref, tmp):
    import torch
    from cape_b200 import demos as ours
    from oracle import tf1_shim as S
    calls, writes = [], []

    class Body(object):
        def __init__(self, faces):
            self.v_template = torch.zeros(6890, 3)
            self.body_pose = torch.zeros(1, 69)
            self.global_orient = torch.zeros(1, 3)
            self.faces = faces

        def __call__(self):
            calls.append((self.v_template.numpy()[::VSTRIDE].copy(), self.global_orient.numpy().ravel().copy(),
                           self.body_pose.numpy().ravel().copy()))
            out = standin_pose(self.v_template.numpy(), self.global_orient.numpy(), self.body_pose.numpy())
            return types.SimpleNamespace(vertices=torch.from_numpy(out[None]))

    class Mesh(object):
        def __init__(self, v=None, f=None, filename=None):
            if filename is not None:
                v, f = ours.read_obj(filename)
            self.v, self.f = v, f

        def write_obj(self, path):
            writes.append((path, np.asarray(self.v, np.float32).reshape(-1, 3)[::VSTRIDE].copy(), len(calls) - 1))

    with H._stubs():
        S.install()
        template = os.path.join(ref, "data", "template_mesh.obj")
        faces = ours.read_obj(template)[1]
        smplx = types.ModuleType("smplx")
        smplx.body_models = types.SimpleNamespace(create=lambda **k: Body(faces))
        sys.modules["smplx"] = smplx
        pm = types.ModuleType("psbody.mesh")
        pm.Mesh = Mesh
        pm.MeshViewers = None
        sys.modules["psbody"] = types.ModuleType("psbody")
        sys.modules["psbody"].mesh = pm
        sys.modules["psbody.mesh"] = pm
        scratch = os.path.join(tmp, "ref")
        os.makedirs(scratch)
        os.symlink(os.path.join(ref, "data"), os.path.join(scratch, "data"))
        spec = importlib.util.spec_from_file_location("ref_demos", os.path.join(ref, "demos.py"))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        mod.__file__ = os.path.join(scratch, "demos.py")
        model = DemoModel()
        with contextlib.redirect_stdout(io.StringIO()):
            demo = mod.demo_full(model, "run", "male", "dset", "unused", "unused", n_sample=N_SAMPLE, save_obj=True,
                                 smpl_model_folder="unused", random_seed=123, vis=False)
            demo.run()
            demo.n_sample = TEST_N_SAMPLE
            demo.test_model(body_data())
        from lib import utils as RU
        from cape_b200 import topology
        rot, pose = topology.demo_pose_params()
        near_pose, near_rot = near_rotations()
        utils = {"utils/rot2pose_demo": RU.rot2pose(rot), "utils/pose2rot_demo": RU.pose2rot(pose),
                 "utils/near_pose": near_pose, "utils/near_rot": near_rot,
                 "utils/pose2rot_near": RU.pose2rot(near_pose), "utils/rot2pose_near": RU.rot2pose(near_rot)}
    res = demo.results_dir
    written = np.zeros(len(calls), bool)
    written[[w[2] for w in writes]] = True
    rec = {"decode/z": np.stack([c[0] for c in model.decode_calls]),
           "decode/cond": np.stack([c[1] for c in model.decode_calls]),
           "decode/cond2": np.stack([c[2] for c in model.decode_calls]),
           "body/v": np.stack([c[0] for c in calls]), "body/global_orient": np.stack([c[1] for c in calls]),
           "body/body_pose": np.stack([c[2] for c in calls]), "body/written": written,
           "obj/paths": np.array([os.path.relpath(w[0], res) for w in writes]),
           "obj/verts": np.stack([w[1] for w in writes]),
           "test/string": np.array(open(os.path.join(res, "test_results_dset.txt")).read()),
           "test/all_file": np.array(open(os.path.join(res, "..", "all_test_results_dset.txt")).read())}
    rec.update(utils)
    return rec


def main():
    import tempfile
    import make_ref_golden as G
    if not os.path.isdir(os.path.join(G.REF, "lib")):
        sys.exit("set CAPE_REFERENCE to a checkout of qianlim/CAPE")
    with tempfile.TemporaryDirectory() as tmp:
        rec = ref_demo_full(G.REF, tmp)
    np.savez_compressed(OUT, **rec)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
