"""SMPL posing on the GPU (cape_smpl_pose) against the float64 oracle, and the test / demo modes of main end to end:
TensorFlow-format checkpoint, synthetic SMPL pickle and dataset in, OBJ files and error statistics out, checked against
the oracle's decoder followed by the oracle's posing."""
import os

import numpy as np
import pytest
import scipy.sparse as sp
import torch

import parity
from test_demo_full import SMPL_PARENTS, synthetic_smpl, write_pickle

pytestmark = pytest.mark.gpu


def _oracle_model(m):
    return {"J_regressor": sp.csr_matrix(m["J_regressor"]), "posedirs": m["posedirs"], "weights": m["weights"],
            "parents": np.array(SMPL_PARENTS)}


def _poses(N, rng):
    """Zero pose, the six shipped demo poses, then random axis-angle vectors with angles up to pi."""
    from cape_b200 import topology as T
    axes = rng.normal(size=(max(N, 7), 24, 3))
    axes /= np.linalg.norm(axes, axis=-1, keepdims=True)
    poses = (axes * rng.uniform(0, np.pi, size=(max(N, 7), 24, 1))).reshape(-1, 72)
    poses[0] = 0
    poses[1:7] = T.demo_pose_params()[1]
    return poses[:N] if N > 1 else poses[1:2]


@pytest.mark.parametrize("N", [1, 7, 64])
def test_posing_kernels_match_the_oracle(N):
    from cape_b200.smpl import SMPL
    from oracle import smpl_lbs
    m = synthetic_smpl(11)
    model = {"v_template": m["v_template"], "f": m["f"], "posedirs": m["posedirs"], "weights": m["weights"],
             "J_regressor": sp.csr_matrix(m["J_regressor"]), "parents": np.array(SMPL_PARENTS)}
    body = SMPL(model)
    rng = np.random.RandomState(N)
    verts = m["v_template"][None] + rng.normal(size=(N, len(m["v_template"]), 3)) * 0.01     # clothed meshes
    poses = _poses(N, rng)
    got = body.pose(verts, poses)
    want = smpl_lbs.lbs_batch(verts.astype(np.float32), poses.astype(np.float32), _oracle_model(m))
    err = np.abs(got - want).max()
    scale = np.abs(want).max()
    print("N=%d: max abs error %.3e (max |v| %.3f, ratio %.2e)" % (N, err, scale, err / scale))
    assert err <= 1e-4 * scale
    if N == 7:      # the zero pose returns the mesh
        assert np.abs(got[0] - verts[0]).max() <= 1e-4 * scale


def test_bad_kinematic_tree_is_refused():
    from cape_b200 import _lib
    from cape_b200.smpl import SMPL
    m = synthetic_smpl(12, V=100)
    parents = np.array(SMPL_PARENTS)
    parents[5] = 7
    with pytest.raises(_lib.CapeError, match="parents"):
        SMPL({"v_template": m["v_template"], "f": m["f"], "posedirs": m["posedirs"], "weights": m["weights"],
              "J_regressor": sp.csr_matrix(m["J_regressor"]), "parents": parents})


# ---- main --mode demo / --mode test ------------------------------------------------------------------------------
YAML = ("nz: 64\nnz_cond: 32\nnz_cond2: 32\naffine: 1\nlr_warmup: 1\nname: e2e\nbatch_size: 4\ndataset: synth\n"
        "pose_type: rot\ndemo_n_sample: 2\nsave_obj: 1\nvis_demo: 0\ngender: male\nsmpl_model_folder: body_models\n")


def _setup(hierarchy, tmp_path):
    from cape_b200 import tf_checkpoint
    from cape_b200.config_parser import model_params, parse_config
    from cape_b200.models import CAPE
    cfg = tmp_path / "c.yaml"
    cfg.write_text(YAML)
    args, _ = parse_config(["--config", str(cfg)])
    p = model_params(args)
    p["p"] = hierarchy["p"]
    h = hierarchy
    m = CAPE(L=h["L"], D=h["D"], U=h["U"], L_d=h["L_d"], D_d=h["D_d"], **p)
    m.build_graph(m.input_num_verts, m.nn_input_channel, phase="demo")
    params = parity.calibrated_params(m.net.specs, 21)
    tf_checkpoint.write_checkpoint(str(tmp_path / "checkpoints" / "e2e" / "model.ckpt-777"),
                                   dict(params, global_step=np.asarray(777, np.int64)))
    smpl_model = synthetic_smpl(13)
    write_pickle(tmp_path / "body_models", "male", smpl_model)
    return str(cfg), m.cfg, params, smpl_model


def _dataset(tmp_path, n_train=110, n_test=6):
    from cape_b200 import smpl
    rng = np.random.RandomState(2)
    d = tmp_path / "data" / "datasets" / "synth"
    for split, n in (("train", n_train), ("test", n_test)):
        os.makedirs(str(d / split))
        np.save(str(d / split / ("%s_disp.npy" % split)), (rng.normal(size=(n, 6890, 3)) * 0.01).astype(np.float32))
        np.save(str(d / split / ("%s_rot.npy" % split)), smpl.pose2rot(rng.normal(size=(n, 72)) * 0.3))
        np.save(str(d / split / ("%s_clo_label.npy" % split)), np.eye(4)[rng.randint(0, 4, size=n)])
    return str(d)


def _check_obj(path, want):
    from cape_b200.demos import read_obj
    v, _ = read_obj(path)
    err = np.abs(v - want).max()
    assert err <= 1e-4 * np.abs(want).max(), (path, err)
    return err


def test_main_demo_mode_writes_the_oracles_meshes(hierarchy, tmp_path, monkeypatch):
    from cape_b200 import main as M
    from cape_b200 import topology as T
    from cape_b200.demos import filter_cloth_pose
    from oracle import cape_oracle as O
    from oracle import smpl_lbs
    cfg_path, cfg, params, smpl_model = _setup(hierarchy, tmp_path)
    monkeypatch.chdir(tmp_path)
    M.main(["--config", cfg_path, "--mode", "demo"], project_dir=str(tmp_path))
    res = tmp_path / "results" / "e2e"
    # the oracle: condition embeddings, the demo's latent draws, decoder, post-processing, posing
    h = hierarchy
    o = O.Oracle(h["L"], h["D"], h["U"], h["L_d"], h["D_d"], cfg)
    P = {k: torch.from_numpy(v) for k, v in params.items()}
    t = torch.from_numpy
    rot, pose = T.demo_pose_params()
    mean, std = T.trainset_stats()
    tv, _ = T.template_mesh()
    keep = T.clothing_verts_idx()
    om = _oracle_model(smpl_model)

    def full(zt, y, y2):
        pred = o.decoder_cond_vert(t(zt.astype(np.float32)), y, y2, P).numpy() * std + mean
        out = np.zeros_like(pred)
        out[:, keep] = pred[:, keep]
        return out + tv

    np.random.seed(123)
    z1 = np.random.normal(size=(2, 64))
    z2 = np.random.normal(size=(2, 64))
    rot14 = filter_cloth_pose(rot).astype(np.float32)
    y, y2 = o.cond_embeddings(t(rot14), t(np.repeat(np.eye(4, dtype=np.float32)[:1], 6, 0)), P)
    errs = []
    for idx in range(6):
        zt = np.concatenate([z1, np.repeat(y[idx:idx + 1].numpy(), 2, 0), np.repeat(y2[:1].numpy(), 2, 0)], 1)
        want = smpl_lbs.lbs_batch(full(zt, y[idx:idx + 1].repeat(2, 1), y2[:1].repeat(2, 1)), np.repeat(pose[idx:idx + 1], 2, 0), om)
        for i in range(2):
            errs.append(_check_obj(str(res / "sample_vary_pose" / ("pose%d_%04d.obj" % (idx, i))), want[i]))
    yc, y2c = o.cond_embeddings(t(np.repeat(rot14[:1], 4, 0)), t(np.eye(4, dtype=np.float32)), P)
    for i, name in enumerate(["shortlong", "shortshort", "longshort", "longlong"]):
        zt = np.concatenate([z2, np.repeat(yc[:1].numpy(), 2, 0), np.repeat(y2c[i:i + 1].numpy(), 2, 0)], 1)
        want = smpl_lbs.lbs_batch(full(zt, yc[:1].repeat(2, 1), y2c[i:i + 1].repeat(2, 1)), np.repeat(pose[2:3], 2, 0), om)
        for j in range(2):
            errs.append(_check_obj(str(res / "sample_vary_clotype" / ("clotype_%s_%04d.obj" % (name, j))), want[j]))
    print("demo mode: %d meshes, max abs error vs oracle %.3e" % (len(errs), max(errs)))
    assert len(os.listdir(str(res / "sample_vary_pose"))) == 12 and len(os.listdir(str(res / "sample_vary_clotype"))) == 8


def test_main_test_mode_reports_the_oracles_errors(hierarchy, tmp_path, monkeypatch):
    from cape_b200 import main as M
    from cape_b200 import smpl
    from cape_b200 import topology as T
    from oracle import cape_oracle as O
    from oracle import smpl_lbs
    cfg_path, cfg, params, smpl_model = _setup(hierarchy, tmp_path)
    data_dir = _dataset(tmp_path)
    monkeypatch.chdir(tmp_path)
    out = M.main(["--config", cfg_path, "--mode", "test"], project_dir=str(tmp_path))
    bd = M.load_body_data(data_dir, "rot")
    h = hierarchy
    o = O.Oracle(h["L"], h["D"], h["U"], h["L_d"], h["D_d"], cfg)
    P = {k: torch.from_numpy(v) for k, v in params.items()}
    t = torch.from_numpy
    y, y2 = o.cond_embeddings(t(bd.cond1_test), t(bd.cond2_test), P)
    rng = np.random.RandomState(cfg["seed"])                  # predict's noise: one draw per (padded) batch of 4
    eps = np.concatenate([rng.normal(size=(4, 64)), rng.normal(size=(4, 64))]).astype(np.float32)
    pred = np.concatenate([o.generator(t(bd.vertices_test[s]), y[s], y2[s], t(eps[s]), P)[0].numpy()
                           for s in (slice(0, 4), slice(4, 6))])
    pred = pred * bd.std + bd.mean
    gt = bd.vertices_test * bd.std + bd.mean
    keep = T.clothing_verts_idx()
    e = np.sqrt(((pred - gt)[:, keep] ** 2).sum(2))
    for k, v in (("mean", e.mean()), ("std", e.std()), ("median", np.median(e))):
        print("test mode: %s %.6f (oracle %.6f)" % (k, out[k], v))
        assert abs(out[k] - v) <= 1e-4 * abs(v), k
    assert "Eucledian err mean {:.5f}".format(out["mean"]) in out["string"]
    res = tmp_path / "results" / "e2e"
    assert open(str(res / "test_results_synth.txt")).read() == out["string"]
    assert open(str(tmp_path / "results" / "all_test_results_synth.txt")).read() == out["string"]
    # posed exemplars: every int(6 / 2) = 3rd test mesh with its pose (rotation matrices -> axis-angle)
    tv, _ = T.template_mesh()
    fullbody = np.zeros_like(pred)
    fullbody[:, keep] = pred[:, keep]
    fullbody = fullbody + tv
    want = smpl_lbs.lbs_batch(fullbody[::3], smpl.rot2pose(bd.cond1_test_full)[::3], _oracle_model(smpl_model))
    objs = sorted(os.listdir(str(res / "test_reconstruction_objs_synth")))
    assert objs == ["0000.obj", "0001.obj"]
    for i in range(2):
        _check_obj(str(res / "test_reconstruction_objs_synth" / objs[i]), want[i])
