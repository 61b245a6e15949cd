#!/usr/bin/env python
"""Golden vectors of the reference's `--activation` and `--loss` switches.  Runs only where $CAPE_REFERENCE names a
checkout.

The reference's unmodified `lib/models.py` runs on the TensorFlow-1 API shim exactly as in make_ref_golden.py (same
inputs, same packing, same sampling of large tensors as make_ref_golden_resblock.py), with `activation` handed to
models.CAPE as main.py does, for three cases, one training update each at batch 2 and global_step 100, written to
tests/golden/ref_models_golden_5.npz (the two affine cases) and ref_models_golden_6.npz (the default model), so that
each file stays under 1 MB:

  * `affine_tanh_huber`: the affine nz64 family with b1tanh and the Huber loss (delta 0.1);
  * `affine_relu_l2`: the affine nz64 family with b1relu and the mean squared error;
  * `default_tanh_l2`: the reference's default model (residual and conditioned encoder, GroupNorm decoder, reduce_dim 4)
    with b1tanh and the mean squared error.

    python tests/golden/make_ref_golden_options.py          (about a minute)
"""
import os

import numpy as np

import make_ref_golden as G
import make_ref_golden_resblock as G3

# file -> the cases it holds (arrays are keyed "<case>/...")
PARTS = {"ref_models_golden_5.npz": ("affine_tanh_huber", "affine_relu_l2"),
         "ref_models_golden_6.npz": ("default_tanh_l2",)}


def configs():
    from cape_b200.params import DEFAULTS, NZ64_AFFINE
    res = dict(use_res_block=True, cond_encoder=True)
    return (("affine_tanh_huber", dict(NZ64_AFFINE, decay_steps=10, activation="b1tanh", loss="huber"), 2, 100),
            ("affine_relu_l2", dict(NZ64_AFFINE, decay_steps=10, activation="b1relu", loss="l2"), 2, 100),
            ("default_tanh_l2", dict(DEFAULTS, reduce_dim=4, affine=False, lambda_edge=0.0, decay_steps=10,
                                     activation="b1tanh", loss="l2", **res), 2, 100))


def load():
    """The arrays of both files in one dict."""
    z = {}
    for name in PARTS:
        with np.load(os.path.join(G.HERE, name)) as f:
            z.update({k: f[k] for k in f.files})
    return z


def run_reference(cfg, h, params, batch, step):
    """G.run_reference with cfg["activation"] among the keyword arguments of models.CAPE (main.py passes it through
    **model_params; G.reference_kwargs leaves it at the reference's default)."""
    base = G.reference_kwargs
    G.reference_kwargs = lambda c, hh, n, name="golden": dict(base(c, hh, n, name), activation=c["activation"])
    try:
        return G.run_reference(cfg, h, params, batch, step)
    finally:
        G.reference_kwargs = base


def main():
    from cape_b200 import topology as T
    L, D, U, p, L_d, D_d, _ = T.load_graph_mtx(load_for_demo=True)
    h = dict(L=L, D=D, U=U, p=p, L_d=L_d, D_d=D_d)
    store = {}
    for tag, cfg, N, step in configs():
        params, batch = G.inputs(cfg, h, N)
        res = run_reference(cfg, h, params, batch, step)
        print("%s: x_hat %s  recon %.6f edge %.6f latent %.6f gan_g %.6f gan_d %.6f  lr %s  (%d variables)"
              % (tag, res["x_hat"].shape, res["recon"], res["edge"], res["latent"], res["gan_g"], res["gan_d"], res["lr"],
                 len(res["created"])))
        G.pack(tag, res, store)
        for k in [k for k in store if k.startswith(tag + "/") and k.endswith("#full") and store[k].size > G3.FULL_MAX]:
            v = store.pop(k).reshape(-1)
            store[k[:-len("#full")] + "#sample"] = v[G.sample_index(k.split("/", 2)[2][:-len("#full")], v.size)]
    for name, tags in PARTS.items():
        out = os.path.join(G.HERE, name)
        np.savez_compressed(out, **{k: v for k, v in store.items() if k.split("/")[0] in tags})
        print("wrote", out, os.path.getsize(out), "bytes")


if __name__ == "__main__":
    main()
