"""The reference's `--activation b1relu|b1tanh` and `--loss l2|huber` against golden vectors of the reference's own
`lib/models.py` (tests/golden/make_ref_golden_options.py -> ref_models_golden_5.npz and _6.npz).

Three cases at batch 2: the affine nz64 family with b1tanh + Huber and with b1relu + L2, and the reference's default
model (residual and conditioned encoder, GroupNorm decoder) with b1tanh + L2.  The oracle (tests/options_oracle.py) has
to reproduce the reference's update with the bounds tests/test_reference_golden_resblock.py uses, and params.param_specs
its variable inventory: the switches add no variables and rename none."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))

import make_ref_golden as G  # noqa: E402
import make_ref_golden_options as G5  # noqa: E402
import options_oracle as OO  # noqa: E402
import test_reference_golden_resblock as T3  # noqa: E402
from oracle import cape_oracle as O  # noqa: E402

TAGS = ["affine_tanh_huber", "affine_relu_l2", "default_tanh_l2"]


def _case(tag):
    return next((c, n, s) for t, c, n, s in G5.configs() if t == tag)


def _update(h, cfg, params, batch, step, ref_compat):
    o = OO.OptOracle(h["L"], h["D"], h["U"], h["L_d"], h["D_d"], cfg)
    P = {k: torch.from_numpy(np.asarray(v, np.float32)) for k, v in params.items()}
    M = {k: torch.zeros_like(v) for k, v in P.items()}
    tb = {k: torch.from_numpy(v) for k, v in batch.items()}
    from cape_b200 import topology as T
    return O.train_update(o, P, M, tb, step, T.smpl_edges(), ref_compat=ref_compat), P


def _compare(z, tag, params, res, res_d, P):
    assert T3._rel(res["x_hat"].numpy(), z[tag + "/x_hat"]) < 1e-6
    for k in ("recon", "edge", "latent", "gan_g", "gan_d"):
        want = float(z["%s/%s" % (tag, k)])
        assert abs(res[k] - want) <= 1e-6 * abs(want), (k, res[k], want)
    bad = {}
    for name in params:
        src = res_d if name.startswith("discriminator") else res
        T3._check_tensor(z, "%s/grads/%s" % (tag, name), src["grads"][name].numpy(), 2e-5, bad)
        T3._check_tensor(z, "%s/params_after/%s" % (tag, name), P[name].numpy(), 2e-5, bad)
    assert not bad, bad


@pytest.mark.parametrize("tag", TAGS)
def test_oracle_reproduces_the_reference(hierarchy, tag):
    z = G5.load()
    cfg, N, step = _case(tag)
    params, batch = G.inputs(cfg, hierarchy, N)
    res, P = _update(hierarchy, cfg, params, batch, step, True)        # the reference's wiring (lib/models.py:466)
    res_d, _ = _update(hierarchy, cfg, params, batch, step, False)     # the discriminator gradients it discards
    _compare(z, tag, params, res, res_d, P)


@pytest.mark.parametrize("tag", TAGS)
def test_variable_inventory_is_the_references(hierarchy, tag):
    z = G5.load()
    cfg, _, _ = _case(tag)
    specs = T3._specs(cfg, hierarchy)
    assert list(specs) == [n for n in T3._inventory(z, tag) if n in specs]
    assert T3._inventory(z, tag) == {k: tuple(v) for k, v in specs.items()}


def test_the_losses_differ_from_l1(hierarchy):
    """What makes the cases worth having: the switches change the reconstruction loss and the encoder's activations
    (the oracle with the default switches gives other numbers on the same inputs)."""
    z = G5.load()
    cfg, N, step = _case("affine_tanh_huber")
    params, batch = G.inputs(cfg, hierarchy, N)
    base, _ = _update(hierarchy, dict(cfg, activation="b1leakyrelu", loss="l1"), params, batch, step, True)
    assert abs(base["recon"] - float(z["affine_tanh_huber/recon"])) > 1e-3 * abs(base["recon"])
    assert T3._rel(base["x_hat"].numpy(), z["affine_tanh_huber/x_hat"]) > 1e-3


@pytest.mark.parametrize("activation,loss", [("b1relu", "l2"), ("b1tanh", "huber"), ("b1leakyrelu", "l2")])
def test_config_parser_and_cape_accept_the_switches(hierarchy, activation, loss):
    from cape_b200.config_parser import model_params, parse_config
    from cape_b200.models import CAPE
    args, _ = parse_config(["--activation", activation, "--loss", loss, "--mode", "demo"])
    kw = model_params(args)
    assert kw["activation"] == activation and kw["loss"] == loss
    h = hierarchy
    m = CAPE(h["L"], h["D"], h["U"], h["L_d"], h["D_d"], **kw)
    assert m.cfg["activation"] == activation and m.cfg["loss"] == loss


@pytest.mark.parametrize("activation", ["b2relu", "b1sigmoid"])
def test_other_activations_still_raise(hierarchy, activation):
    from cape_b200.config_parser import model_params, parse_config
    from cape_b200.models import CAPE
    args, _ = parse_config(["--activation", activation, "--mode", "demo"])
    h = hierarchy
    with pytest.raises(NotImplementedError, match="activation"):
        CAPE(h["L"], h["D"], h["U"], h["L_d"], h["D_d"], **model_params(args))


def test_loss_kinds_follow_the_reference():
    """models.py:357-369: 'l1', 'huber', and the mean squared error for every other string ('l2' included)."""
    from cape_b200 import engine as E
    assert E.recon_kind("l1") == E.RECON_L1 and E.recon_kind("huber") == E.RECON_HUBER
    assert E.recon_kind("l2") == E.RECON_L2 and E.recon_kind("mse") == E.RECON_L2
    assert E.brelu("b1relu") == (E.ACT_RELU, E.EPI_SLOPE, 0.0)
    assert E.brelu("b1tanh")[:2] == (E.ACT_TANH, E.EPI_TANHGRAD)


def test_default_switches_leave_the_oracle_unchanged(hierarchy):
    """With b1leakyrelu / l1 the oracle of these tests is the residual-encoder oracle, bit for bit."""
    import resblock_oracle as R
    cfg, N, step = _case("default_tanh_l2")
    cfg = dict(cfg, activation="b1leakyrelu", loss="l1")
    params, batch = G.inputs(cfg, hierarchy, 1)
    h = hierarchy
    from cape_b200 import topology as T
    outs = []
    for cls in (R.ResOracle, OO.OptOracle):
        P = {k: torch.from_numpy(np.asarray(v, np.float32)) for k, v in params.items()}
        M = {k: torch.zeros_like(v) for k, v in P.items()}
        tb = {k: torch.from_numpy(v) for k, v in batch.items()}
        outs.append(O.train_update(cls(h["L"], h["D"], h["U"], h["L_d"], h["D_d"], cfg), P, M, tb, step, T.smpl_edges()))
    assert torch.equal(outs[0]["x_hat"], outs[1]["x_hat"])
    assert all(torch.equal(outs[0]["grads"][k], outs[1]["grads"][k]) for k in outs[0]["grads"])


@pytest.mark.skipif(not os.environ.get("CAPE_REFERENCE"), reason="needs $CAPE_REFERENCE (a reference checkout)")
@pytest.mark.parametrize("tag", TAGS)
def test_reference_rerun_matches_the_file(hierarchy, tag):
    """The committed vectors are what the reference computes now (G5.run_reference on the shim)."""
    z = G5.load()
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
