"""The model at layer widths the shipped configurations never use, against golden vectors of the reference's own
`lib/models.py` (tests/golden/make_ref_golden_widths.py -> ref_models_golden_4.npz).

Two cases at batch 2: `affine_nf48` (the affine nz64 family at --nf 48, 27 condition channels, reduce_dim 6) and
`default_nf32` (the reference's default model at --nf 32: GroupNorm blocks of 16 channels).  The oracle has to reproduce
the reference's update with the bounds tests/test_reference_golden_resblock.py uses, and params.param_specs its
variable inventory."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))

import make_ref_golden as G  # noqa: E402
import make_ref_golden_widths as G4  # noqa: E402
import test_reference_golden_resblock as T3  # noqa: E402

TAGS = ["affine_nf48", "default_nf32"]


def _case(tag):
    return next((c, n, s) for t, c, n, s in G4.configs() if t == tag)


@pytest.mark.parametrize("tag", TAGS)
def test_oracle_reproduces_the_reference(hierarchy, tag):
    z = G4.load()
    cfg, N, step = _case(tag)
    params, batch = G.inputs(cfg, hierarchy, N)
    res, P = T3._update(hierarchy, cfg, params, batch, step, True)        # the reference's wiring (lib/models.py:466)
    res_d, _ = T3._update(hierarchy, cfg, params, batch, step, False)     # the discriminator gradients it discards
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
def test_variable_inventory_is_the_references(hierarchy, tag):
    z = G4.load()
    cfg, _, _ = _case(tag)
    specs = T3._specs(cfg, hierarchy)
    assert list(specs) == [n for n in T3._inventory(z, tag) if n in specs]          # the reference's creation order
    assert T3._inventory(z, tag) == {k: tuple(v) for k, v in specs.items()}


def test_widths_are_off_the_shipped_grid(hierarchy):
    """What makes these cases worth having: conv widths that are not multiples of 32, an odd condition width, a 6-wide
    bottleneck (affine_nf48); 16-channel GroupNorm blocks (default_nf32)."""
    cfg, _, _ = _case("affine_nf48")
    specs = T3._specs(cfg, hierarchy)
    assert cfg["nz_cond"] + cfg["nz_cond2"] == 27
    assert specs["generator/encoder/1x1-conv/weights"] == (384, 6)
    assert any(s[-1] % 32 for s in specs.values())
    cfg, _, _ = _case("default_nf32")
    assert cfg["F"] == [32, 32, 64, 64, 128, 128, 256, 256] and cfg["reduce_dim"] == 4
