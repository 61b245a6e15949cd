"""The reference's plain decoder (`--use_res_block_dec 0`) and `--reduce_dim 0` against golden vectors of the reference's
own `lib/models.py` (tests/golden/make_ref_golden_plaindec.py -> ref_models_golden_7.npz and _8.npz).

Four cases at batch 2: the nz18 model with the plain decoder; the nz64 family with the plain decoder, reduce_dim 0,
b1tanh and L2; the reference's default model with reduce_dim 0; and the affine nz64 family with reduce_dim 0 and b1relu.
The oracle (tests/plaindec_oracle.py) has to reproduce the reference's update with the bounds
tests/test_reference_golden_resblock.py uses, and params.param_specs its variable inventory, order included."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))

import make_ref_golden as G  # noqa: E402
import make_ref_golden_options as G5  # noqa: E402
import make_ref_golden_plaindec as G7  # noqa: E402
import options_oracle as OO  # noqa: E402
import plaindec_oracle as PD  # noqa: E402
import test_reference_golden_options as T5  # noqa: E402
import test_reference_golden_resblock as T3  # noqa: E402
from oracle import cape_oracle as O  # noqa: E402

TAGS = ["plain_nz18", "plain_nz64_rd0_tanh_l2", "default_rd0", "affine_rd0_relu"]


def _case(tag):
    return next((c, n, s) for t, c, n, s in G7.configs() if t == tag)


def _update(h, cfg, params, batch, step, ref_compat, cls=PD.PlainDecOracle):
    o = cls(h["L"], h["D"], h["U"], h["L_d"], h["D_d"], cfg)
    P = {k: torch.from_numpy(np.asarray(v, np.float32)) for k, v in params.items()}
    M = {k: torch.zeros_like(v) for k, v in P.items()}
    tb = {k: torch.from_numpy(v) for k, v in batch.items()}
    from cape_b200 import topology as T
    return O.train_update(o, P, M, tb, step, T.smpl_edges(), ref_compat=ref_compat), P


@pytest.mark.parametrize("tag", TAGS)
def test_oracle_reproduces_the_reference(hierarchy, tag):
    z = G7.load()
    cfg, N, step = _case(tag)
    params, batch = G.inputs(cfg, hierarchy, N)
    res, P = _update(hierarchy, cfg, params, batch, step, True)        # the reference's wiring (lib/models.py:466)
    res_d, _ = _update(hierarchy, cfg, params, batch, step, False)     # the discriminator gradients it discards
    T5._compare(z, tag, params, res, res_d, P)


@pytest.mark.parametrize("tag", TAGS)
def test_variable_inventory_is_the_references(hierarchy, tag):
    z = G7.load()
    cfg, _, _ = _case(tag)
    specs = T3._specs(cfg, hierarchy)
    assert list(specs) == [n for n in T3._inventory(z, tag) if n in specs]
    assert T3._inventory(z, tag) == {k: tuple(v) for k, v in specs.items()}


def test_plain_decoder_variables(hierarchy):
    """The shapes the plain decoder adds: [(F_in + Cc) K, F_out] weights and [1, 1, F_out] biases; at reduce_dim 0 the
    FC layers read and write p[-1] F[-1] = 862 x 512 features."""
    specs = T3._specs(_case("plain_nz18")[0], hierarchy)
    assert specs["generator/decoder/decoder_conv1/weights"] == (1088, 512)
    assert specs["generator/decoder/decoder_conv8/weights"] == (192, 64)
    assert specs["generator/decoder/decoder_conv8/bias"] == (1, 1, 64)
    assert specs["generator/decoder/outputs/weights"] == ((64 + 32) * 2, 3)
    assert not any("resblock" in n for n in specs if n.startswith("generator/decoder"))
    specs = T3._specs(_case("plain_nz64_rd0_tanh_l2")[0], hierarchy)
    assert specs["generator/encoder/fc_mean/dense/kernel"] == (441344, 64)
    assert specs["generator/decoder/fc1/dense/kernel"] == (128, 441344)
    assert not any("1x1-conv" in n for n in specs)


def test_residual_decoder_leaves_the_oracle_unchanged(hierarchy):
    """With use_res_block_dec on, the oracle of these tests is the options oracle: the same forward bit for bit, the same
    gradients up to the order in which torch's CPU threads add the 441 344-long reductions of the FC layers."""
    cfg, _, step = _case("affine_rd0_relu")
    params, batch = G.inputs(cfg, hierarchy, 1)
    outs = [_update(hierarchy, cfg, params, batch, step, False, cls)[0] for cls in (OO.OptOracle, PD.PlainDecOracle)]
    assert torch.equal(outs[0]["x_hat"], outs[1]["x_hat"])
    assert all(T3._rel(outs[1]["grads"][k].numpy(), outs[0]["grads"][k].numpy()) < 1e-6 for k in outs[0]["grads"])


@pytest.mark.parametrize("tag", ["plain_nz18", "affine_rd0_relu"])
def test_cape_builds_the_switches(hierarchy, tag):
    """The config parser's switches reach CAPE, which builds its parameter inventory without refusing."""
    from cape_b200.config_parser import model_params, parse_config
    from cape_b200.models import CAPE
    cfg, _, _ = _case(tag)
    argv = ["--mode", "demo", "--use_res_block_dec", str(int(cfg["use_res_block_dec"])),
            "--reduce_dim", str(cfg["reduce_dim"])]
    kw = model_params(parse_config(argv)[0])
    h = hierarchy
    m = CAPE(h["L"], h["D"], h["U"], h["L_d"], h["D_d"], **kw)
    assert bool(m.cfg["use_res_block_dec"]) == bool(cfg["use_res_block_dec"])
    assert m.cfg["reduce_dim"] == cfg["reduce_dim"]


@pytest.mark.skipif(not os.environ.get("CAPE_REFERENCE"), reason="needs $CAPE_REFERENCE (a reference checkout)")
@pytest.mark.parametrize("tag", TAGS)
def test_reference_rerun_matches_the_file(hierarchy, tag):
    """The committed vectors are what the reference computes now (on the shim)."""
    z = G7.load()
    cfg, N, step = _case(tag)
    params, batch = G.inputs(cfg, hierarchy, N)
    res = G5.run_reference(cfg, hierarchy, params, batch, step)
    store = {}
    G.pack(tag, res, store)
    assert np.array_equal(res["x_hat"], z[tag + "/x_hat"])
    for k in ("recon", "edge", "latent", "gan_g", "gan_d"):
        assert float(store["%s/%s" % (tag, k)]) == float(z["%s/%s" % (tag, k)])
    for k, v in store.items():
        if k.endswith("#l2"):
            assert abs(float(v) - float(z[k])) <= 1e-6 * max(float(z[k]), 1e-30), k
