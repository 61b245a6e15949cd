#!/usr/bin/env python
"""Golden vectors of the reference's `--loss_mask binary`.  Runs only where $CAPE_REFERENCE names a checkout.

The reference's unmodified `lib/models.py` runs on the TensorFlow-1 API shim exactly as in make_ref_golden_options.py
(same inputs, same packing, same sampling of large tensors, `activation` handed to models.CAPE), for three cases, one
training update each at batch 2 and global_step 100, written to tests/golden/ref_models_golden_9.npz and
ref_models_golden_10.npz so that each file stays under 1 MB:

  * `affine_l1_mask`: the affine nz64 family with the L1 loss;
  * `nz18_l2_mask`: the nz18 GroupNorm family with the mean squared error;
  * `default_huber_mask`: the reference's default model (residual and conditioned encoder, GroupNorm decoder,
    reduce_dim 4) with the Huber loss (delta 0.1).

One step departs from the reference's path.  models.CAPE is built with loss_mask=None, and before `build_graph` the
script sets `model.loss_mask = np.repeat(m[None, :, None], N, 0)`, the [N, 6890, 1] array `loss()` hands to every
reconstruction loss as `weights` (models.py:357-369).  The reference cannot build that array itself with
`loss_mask='binary'`: it looks for the mask in lib/data/ (models.py:49), and the file it ships, data/loss_mask_binary.npy,
is 1-D while models.py:50 indexes it as 2-D.  The array set here is what that line gives for a [6890, 1] file.  m is
the float32 copy of the shipped file that the package trains with (tests/golden/loss_mask_binary.npz).

    python tests/golden/make_ref_golden_lossmask.py          (about a minute)
"""
import os

import numpy as np

import make_ref_golden as G
import make_ref_golden_options as G5
import make_ref_golden_resblock as G3

# file -> the cases it holds (arrays are keyed "<case>/...")
PARTS = {"ref_models_golden_9.npz": ("affine_l1_mask", "nz18_l2_mask"),
         "ref_models_golden_10.npz": ("default_huber_mask",)}


def configs():
    from cape_b200.params import DEFAULTS, NZ18_PLAIN, NZ64_AFFINE
    res = dict(use_res_block=True, cond_encoder=True)
    return (("affine_l1_mask", dict(NZ64_AFFINE, decay_steps=10, loss="l1", loss_mask="binary"), 2, 100),
            ("nz18_l2_mask", dict(NZ18_PLAIN, decay_steps=10, loss="l2", loss_mask="binary"), 2, 100),
            ("default_huber_mask", dict(DEFAULTS, reduce_dim=4, affine=False, lambda_edge=0.0, decay_steps=10,
                                        loss="huber", loss_mask="binary", **res), 2, 100))


def load():
    """The arrays of both files in one dict."""
    z = {}
    for name in PARTS:
        with np.load(os.path.join(G.HERE, name)) as f:
            z.update({k: f[k] for k in f.files})
    return z


def run_reference(cfg, h, params, batch, step):
    """G5.run_reference with the reference's `self.loss_mask` set to the [N, 6890, 1] weights before build_graph."""
    from oracle import tf1_shim as S
    from cape_b200 import topology as T
    S.install(template_vertices=T.template_mesh()[0])
    from lib import models as RM                                 # the reference's own module
    N = batch["x_g"].shape[0]
    weights = np.repeat(T.loss_mask_binary()[None, :, None], N, 0)
    build = RM.CAPE.build_graph

    def build_masked(model, *a, **k):
        model.loss_mask = weights
        return build(model, *a, **k)

    RM.CAPE.build_graph = build_masked
    try:
        return G5.run_reference(cfg, h, params, batch, step)
    finally:
        RM.CAPE.build_graph = build


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
