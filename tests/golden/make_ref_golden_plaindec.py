#!/usr/bin/env python
"""Golden vectors of the reference's plain decoder (`--use_res_block_dec 0`) and of `--reduce_dim 0`.  Runs only where
$CAPE_REFERENCE names a checkout.

The reference's unmodified `lib/models.py` runs on the TensorFlow-1 API shim exactly as in make_ref_golden_options.py
(same inputs, same packing, same sampling of large tensors, `activation` handed to models.CAPE), for four cases, one
training update each at batch 2 and global_step 100, written to tests/golden/ref_models_golden_7.npz and
ref_models_golden_8.npz so that each file stays under 1 MB:

  * `plain_nz18`: DEFAULTS with the plain decoder (udn, models.py:173-191);
  * `plain_nz64_rd0_tanh_l2`: the nz64 family (nz 64, nz_cond 32, nz_cond2 32) with the plain decoder, reduce_dim 0,
    b1tanh and the mean squared error -- `affine` is left on, and the plain decoder wins (models.py:597-603);
  * `default_rd0`: the reference's default model (residual and conditioned encoder, GroupNorm decoder) with reduce_dim 0:
    the residual encoder feeds the FC layers, and fc1 feeds the GroupNorm decoder;
  * `affine_rd0_relu`: the affine nz64 family with reduce_dim 0 and b1relu.

    python tests/golden/make_ref_golden_plaindec.py          (a few minutes)
"""
import os

import numpy as np

import make_ref_golden as G
import make_ref_golden_options as G5
import make_ref_golden_resblock as G3

# file -> the cases it holds (arrays are keyed "<case>/...")
PARTS = {"ref_models_golden_7.npz": ("plain_nz18", "plain_nz64_rd0_tanh_l2"),
         "ref_models_golden_8.npz": ("default_rd0", "affine_rd0_relu")}


def configs():
    from cape_b200.params import DEFAULTS, NZ64_AFFINE
    res = dict(use_res_block=True, cond_encoder=True)
    return (("plain_nz18", dict(DEFAULTS, use_res_block_dec=False, decay_steps=10), 2, 100),
            ("plain_nz64_rd0_tanh_l2", dict(NZ64_AFFINE, use_res_block_dec=False, reduce_dim=0, decay_steps=10,
                                            activation="b1tanh", loss="l2"), 2, 100),
            ("default_rd0", dict(DEFAULTS, reduce_dim=0, affine=False, lambda_edge=0.0, decay_steps=10, **res), 2, 100),
            ("affine_rd0_relu", dict(NZ64_AFFINE, reduce_dim=0, decay_steps=10, activation="b1relu"), 2, 100))


def load():
    """The arrays of both files in one dict."""
    z = {}
    for name in PARTS:
        with np.load(os.path.join(G.HERE, name)) as f:
            z.update({k: f[k] for k in f.files})
    return z


def main():
    from cape_b200 import topology as T
    L, D, U, p, L_d, D_d, _ = T.load_graph_mtx(load_for_demo=True)
    h = dict(L=L, D=D, U=U, p=p, L_d=L_d, D_d=D_d)
    store = {}
    for tag, cfg, N, step in configs():
        params, batch = G.inputs(cfg, h, N)
        res = G5.run_reference(cfg, h, params, batch, step)
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
