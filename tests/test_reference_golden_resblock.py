"""The reference's default encoder -- residual encoder blocks and the conditioned encoder -- against golden vectors of
the reference's own `lib/models.py` (tests/golden/make_ref_golden_resblock.py -> ref_models_golden_3.npz).

Two cases: `default` (configs/default_config.yaml: GroupNorm decoder, reduce_dim 4, batch 1) and `res_affine` (the
affine-decoder nz64 family with the same encoder, batch 2).  The oracle (tests/resblock_oracle.py) has to reproduce the
reference's update with the bounds tests/test_reference_golden.py uses, and params.param_specs its variable inventory."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))

import make_host_golden as H  # noqa: E402
import make_ref_golden as G  # noqa: E402
import make_ref_golden_resblock as G3  # noqa: E402
import resblock_oracle as R  # noqa: E402
from oracle import cape_oracle as O  # noqa: E402


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def _check_tensor(z, base, v, tol, bad):
    v = np.asarray(v, np.float32)
    l2 = np.sqrt((v.astype(np.float64) ** 2).sum())
    want = float(z[base + "#l2"])
    if abs(l2 - want) > tol * max(want, 1e-30):
        bad[base + "#l2"] = (l2, want)
    if base + "#full" in z:
        e = _rel(v, z[base + "#full"])
    else:
        e = _rel(v.reshape(-1)[G.sample_index(base.split("/", 2)[2], v.size)], z[base + "#sample"])
    if not e < tol:
        bad[base] = e


def _case(tag):
    return next((c, n, s) for t, c, n, s in G3.configs() if t == tag)


def _update(h, cfg, params, batch, step, ref_compat):
    o = R.ResOracle(h["L"], h["D"], h["U"], h["L_d"], h["D_d"], cfg)
    P = {k: torch.from_numpy(np.asarray(v, np.float32)) for k, v in params.items()}
    M = {k: torch.zeros_like(v) for k, v in P.items()}
    tb = {k: torch.from_numpy(v) for k, v in batch.items()}
    from cape_b200 import topology as T
    return O.train_update(o, P, M, tb, step, T.smpl_edges(), ref_compat=ref_compat), P


def _specs(cfg, h):
    from cape_b200.params import param_specs
    return param_specs(cfg, [l.shape[0] for l in h["L"]], [l.shape[0] for l in h["L_d"]])


def _inventory(z, tag):
    return {str(n): tuple(int(x) for x in str(s).split(",")) for n, s in zip(z[tag + "/var_names"], z[tag + "/var_shapes"])}


@pytest.mark.parametrize("tag", ["default", "res_affine"])
def test_oracle_reproduces_the_reference(hierarchy, tag):
    z = G3.load()
    cfg, N, step = _case(tag)
    params, batch = G.inputs(cfg, hierarchy, N)
    res, P = _update(hierarchy, cfg, params, batch, step, True)        # the reference's wiring (lib/models.py:466)
    res_d, _ = _update(hierarchy, cfg, params, batch, step, False)     # the discriminator gradients it discards
    assert _rel(res["x_hat"].numpy(), z[tag + "/x_hat"]) < 1e-6
    for k in ("recon", "edge", "latent", "gan_g", "gan_d"):
        want = float(z["%s/%s" % (tag, k)])
        assert abs(res[k] - want) <= 1e-6 * abs(want), (k, res[k], want)
    bad = {}
    for name in params:
        src = res_d if name.startswith("discriminator") else res
        _check_tensor(z, "%s/grads/%s" % (tag, name), src["grads"][name].numpy(), 2e-5, bad)
        _check_tensor(z, "%s/params_after/%s" % (tag, name), P[name].numpy(), 2e-5, bad)
    assert not bad, bad


@pytest.mark.parametrize("tag", ["default", "res_affine"])
def test_variable_inventory_is_the_references(hierarchy, tag):
    z = G3.load()
    cfg, _, _ = _case(tag)
    specs = _specs(cfg, hierarchy)
    assert list(specs) == [n for n in _inventory(z, tag) if n in specs]          # the reference's creation order
    assert _inventory(z, tag) == {k: tuple(v) for k, v in specs.items()}


def test_residual_blocks_project_where_the_channel_count_changes(hierarchy):
    """Blocks 1, 3, 5 and 7 have a 1x1 projection on the skip (block 1 over the 3 + 32 conditioned input channels);
    2, 4, 6 and 8 add their input unchanged."""
    cfg, _, _ = _case("default")
    specs = _specs(cfg, hierarchy)
    proj = {i for i in range(1, 9) if "generator/encoder/encoder_resblock%d/1x1-conv/weights" % i in specs}
    assert proj == {1, 3, 5, 7}
    assert specs["generator/encoder/encoder_resblock1/filter_1/weights"] == (70, 64)
    assert specs["generator/encoder/encoder_resblock1/1x1-conv/weights"] == (35, 64)
    assert specs["generator/encoder/1x1-conv/weights"] == (512, 4)


def test_oracle_reproduces_the_reference_demo_graph(hierarchy):
    """op_vae_mean / op_vae_var see the condition embeddings; op_decoder is the GroupNorm decoder."""
    z = G3.load()
    tag = "default"
    cfg, N, _ = _case(tag)
    params, batch = G.inputs(cfg, hierarchy, N)
    df = G.demo_feeds(cfg, N)
    h = hierarchy
    o = R.ResOracle(h["L"], h["D"], h["U"], h["L_d"], h["D_d"], cfg)
    P = {k: torch.from_numpy(v) for k, v in params.items()}
    t = torch.from_numpy
    with torch.no_grad():
        dec = o.decoder_cond_vert(t(df["z_total"]), t(df["cond_latent"]), t(df["cond2_latent"]), P)
        y, y2 = o.cond_embeddings(t(batch["cond_g"]), t(batch["cond2_g"]), P)
        zm, zl = o.encoder(t(batch["x_g"]), P, y, y2)
    assert _rel(dec.numpy(), z[tag + "/demo/decoded"]) < 1e-6
    assert _rel(zm.numpy(), z[tag + "/demo/vae_mean"]) < 1e-6 and _rel(zl.numpy(), z[tag + "/demo/vae_var"]) < 1e-6
    assert _rel(y.numpy(), z[tag + "/demo/cond_latent"]) < 1e-6 and _rel(y2.numpy(), z[tag + "/demo/cond2_latent"]) < 1e-6


def test_default_config_yaml_builds_the_references_inventory(hierarchy, tmp_path):
    """The reference's configs/default_config.yaml, parsed like a user's --config, yields the variables the reference
    created for its default model."""
    from cape_b200.config_parser import model_params, parse_config
    from cape_b200.params import DEFAULTS
    cfgs = np.load(H.CONFIGS_OUT)
    texts = dict(zip(cfgs["names"].tolist(), cfgs["texts"].tolist()))
    yml = tmp_path / "default_config.yaml"
    yml.write_text(texts["default_config.yaml"])
    args, _ = parse_config(["--config", str(yml), "--mode", "demo"])
    kw = model_params(args)
    cfg = dict(DEFAULTS, **{k: v for k, v in kw.items() if k in DEFAULTS})
    assert cfg["use_res_block"] and cfg["cond_encoder"] and cfg["reduce_dim"] == 4 and not cfg["affine"]
    assert _inventory(G3.load(), "default") == {k: tuple(v) for k, v in _specs(cfg, hierarchy).items()}


def test_plain_configurations_keep_their_inventory(hierarchy):
    """Without use_res_block / cond_encoder, param_specs and the oracle's encoder are what they were."""
    z = G.load()
    for tag in ("nz64", "nz18"):
        cfg = next(c for t, c, n, s in G.configs() if t == tag)
        assert _inventory(z, tag) == {k: tuple(v) for k, v in _specs(cfg, hierarchy).items()}
        params, batch = G.inputs(cfg, hierarchy, 1)
        h = hierarchy
        P = {k: torch.from_numpy(v) for k, v in params.items()}
        x = torch.from_numpy(batch["x_g"])
        with torch.no_grad():
            a = R.ResOracle(h["L"], h["D"], h["U"], h["L_d"], h["D_d"], cfg).encoder(x, P)
            b = O.Oracle(h["L"], h["D"], h["U"], h["L_d"], h["D_d"], cfg).encoder(x, P)
        assert all(torch.equal(u, v) for u, v in zip(a, b))
