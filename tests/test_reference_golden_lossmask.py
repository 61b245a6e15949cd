"""The reference's `--loss_mask binary` against golden vectors of the reference's own `lib/models.py`
(tests/golden/make_ref_golden_lossmask.py -> ref_models_golden_9.npz and _10.npz).

Three cases at batch 2: the affine nz64 family with L1, the nz18 GroupNorm family with L2, and the reference's default
model (residual and conditioned encoder, GroupNorm decoder) with Huber, each with the shipped per-vertex mask on the
reconstruction term.  The oracle (tests/lossmask_oracle.py) has to reproduce the reference's update with the bounds of
tests/test_reference_golden_options.py.  The fixture tests/golden/loss_mask_binary.npz is the reference's
data/loss_mask_binary.npy, and every `loss_mask` value other than 'binary' means no mask (models.py:47-52)."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))

import make_ref_golden as G  # noqa: E402
import make_ref_golden_lossmask as G9  # noqa: E402
import lossmask_oracle as LM  # noqa: E402
import options_oracle as OO  # noqa: E402
import test_reference_golden_options as T5  # noqa: E402
import test_reference_golden_resblock as T3  # noqa: E402
from oracle import cape_oracle as O  # noqa: E402

TAGS = ["affine_l1_mask", "nz18_l2_mask", "default_huber_mask"]


def _case(tag):
    return next((c, n, s) for t, c, n, s in G9.configs() if t == tag)


def _update(h, cfg, params, batch, step, ref_compat, cls=LM.MaskOracle):
    o = cls(h["L"], h["D"], h["U"], h["L_d"], h["D_d"], cfg)
    P = {k: torch.from_numpy(np.asarray(v, np.float32)) for k, v in params.items()}
    M = {k: torch.zeros_like(v) for k, v in P.items()}
    tb = {k: torch.from_numpy(v) for k, v in batch.items()}
    from cape_b200 import topology as T
    return O.train_update(o, P, M, tb, step, T.smpl_edges(), ref_compat=ref_compat), P


@pytest.mark.parametrize("tag", TAGS)
def test_oracle_reproduces_the_reference(hierarchy, tag):
    z = G9.load()
    cfg, N, step = _case(tag)
    params, batch = G.inputs(cfg, hierarchy, N)
    res, P = _update(hierarchy, cfg, params, batch, step, True)        # the reference's wiring (lib/models.py:466)
    res_d, _ = _update(hierarchy, cfg, params, batch, step, False)     # the discriminator gradients it discards
    T5._compare(z, tag, params, res, res_d, P)


@pytest.mark.parametrize("tag", TAGS)
def test_variable_inventory_is_the_references(hierarchy, tag):
    """The mask is not a variable: the inventory is the unmasked model's."""
    z = G9.load()
    cfg, _, _ = _case(tag)
    specs = T3._specs(cfg, hierarchy)
    assert list(specs) == [n for n in T3._inventory(z, tag) if n in specs]
    assert T3._inventory(z, tag) == {k: tuple(v) for k, v in specs.items()}


@pytest.mark.parametrize("tag", TAGS)
def test_the_mask_changes_the_update(hierarchy, tag):
    """What makes the cases worth having: without the mask the oracle gives another reconstruction term and other
    generator gradients on the same inputs, while x_hat and the edge term stay the same."""
    z = G9.load()
    cfg, N, step = _case(tag)
    params, batch = G.inputs(cfg, hierarchy, N)
    base, _ = _update(hierarchy, dict(cfg, loss_mask=None), params, batch, step, True)
    assert abs(base["recon"] - float(z[tag + "/recon"])) > 1e-4 * abs(base["recon"])     # 100x the test bound
    assert T3._rel(base["x_hat"].numpy(), z[tag + "/x_hat"]) < 1e-6
    assert abs(base["edge"] - float(z[tag + "/edge"])) <= 1e-6 * float(z[tag + "/edge"])
    name = "generator/decoder/outputs/bias"
    g = base["grads"][name].numpy().reshape(-1)
    assert T3._rel(g[G.sample_index(name, g.size)], z["%s/grads/%s#sample" % (tag, name)]) > 1e-2


def test_fixture_is_the_shipped_mask():
    from cape_b200 import topology as T
    m = T.loss_mask_binary()
    assert m.dtype == np.float32 and m.shape == (6890,)
    assert np.array_equal(np.unique(m), np.float32([0.1, 1.0]))
    assert int((m == 1.0).sum()) == 4425                    # 4425 + 0.1 * 2465 = 4671.5


@pytest.mark.skipif(not os.environ.get("CAPE_REFERENCE"), reason="needs $CAPE_REFERENCE (a reference checkout)")
def test_fixture_equals_the_references_file():
    from cape_b200 import topology as T
    ref = np.load(os.path.join(os.environ["CAPE_REFERENCE"], "data", "loss_mask_binary.npy"))
    assert ref.shape == (6890,)
    assert np.array_equal(T.loss_mask_binary(), ref.astype(np.float32))


def _cape(h, argv):
    from cape_b200.config_parser import model_params, parse_config
    from cape_b200.models import CAPE
    args, _ = parse_config(argv + ["--mode", "demo"])
    return CAPE(h["L"], h["D"], h["U"], h["L_d"], h["D_d"], **model_params(args)), args


def test_config_parser_and_cape_accept_binary(hierarchy):
    m, args = _cape(hierarchy, ["--loss_mask", "binary"])
    assert args.loss_mask == "binary" and m.cfg["loss_mask"] == "binary"


@pytest.mark.parametrize("value", ["", "None", "Binary", "clothing"])
def test_other_values_build_unmasked_models(hierarchy, value):
    """models.py:47-52: only the string 'binary' selects the mask; '' (the parser's default), the string 'None' of
    configs/default_config.yaml and any other string mean weights 1.0."""
    m, args = _cape(hierarchy, ["--loss_mask", value])
    assert args.loss_mask == value and m.cfg["loss_mask"] is None


def test_loss_mask_none_builds_an_unmasked_model(hierarchy):
    from cape_b200.models import CAPE
    cfg, _, _ = _case("affine_l1_mask")
    h = hierarchy
    m = CAPE(**dict(G.reference_kwargs(cfg, dict(h, p=h["p"]), 2), loss_mask=None))
    assert m.cfg["loss_mask"] is None


def test_b2relu_still_raises_with_the_mask(hierarchy):
    with pytest.raises(NotImplementedError, match="activation"):
        _cape(hierarchy, ["--loss_mask", "binary", "--activation", "b2relu"])


@pytest.mark.parametrize("loss", ["l1", "l2", "huber"])
def test_oracle_reconstruction_term(hierarchy, loss):
    """MaskOracle.recon_loss: OptOracle's without 'binary'; with it, sum m[v] l(d) / (3 N sum m) in float64."""
    from cape_b200 import topology as T
    h = hierarchy
    d = torch.from_numpy(np.random.RandomState(1).normal(0, 0.2, size=(2, 6890, 3)))
    cfg, _, _ = _case("affine_l1_mask")
    plain = OO.OptOracle(h["L"], h["D"], h["U"], h["L_d"], h["D_d"], dict(cfg, loss=loss, loss_mask=""))
    for value in ("", None, "other"):
        o = LM.MaskOracle(h["L"], h["D"], h["U"], h["L_d"], h["D_d"], dict(cfg, loss=loss, loss_mask=value))
        assert float(o.recon_loss(d)) == float(plain.recon_loss(d))
    o = LM.MaskOracle(h["L"], h["D"], h["U"], h["L_d"], h["D_d"], dict(cfg, loss=loss))
    m = T.loss_mask_binary().astype(np.float64)
    x = d.numpy()
    q = np.minimum(np.abs(x), 0.1)
    ell = {"l1": np.abs(x), "l2": x * x, "huber": 0.5 * q * q + 0.1 * (np.abs(x) - q)}[loss]
    want = (ell * m[None, :, None]).sum() / (3 * 2 * m.sum())
    assert abs(float(o.recon_loss(d)) - want) <= 1e-12 * want


@pytest.mark.skipif(not os.environ.get("CAPE_REFERENCE"), reason="needs $CAPE_REFERENCE (a reference checkout)")
@pytest.mark.parametrize("tag", TAGS)
def test_reference_rerun_matches_the_file(hierarchy, tag):
    """The committed vectors are what the reference computes now (G9.run_reference on the shim)."""
    z = G9.load()
    cfg, N, step = _case(tag)
    params, batch = G.inputs(cfg, hierarchy, N)
    res = G9.run_reference(cfg, hierarchy, params, batch, step)
    store = {}
    G.pack(tag, res, store)
    assert np.array_equal(res["x_hat"], z[tag + "/x_hat"])
    for k in ("recon", "edge", "latent", "gan_g", "gan_d"):
        assert float(store["%s/%s" % (tag, k)]) == float(z["%s/%s" % (tag, k)])
