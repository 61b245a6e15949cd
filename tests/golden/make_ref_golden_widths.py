#!/usr/bin/env python
"""Golden vectors of the reference at layer widths the shipped configurations never use.  Runs only where
$CAPE_REFERENCE names a checkout.

The reference's unmodified `lib/models.py` runs on the TensorFlow-1 API shim exactly as in make_ref_golden.py (same
inputs, same packing, same sampling of large tensors as make_ref_golden_resblock.py) for two cases, one training update
each at batch 2 and global_step 100, written to tests/golden/ref_models_golden_4.npz:

  * `affine_nf48`: the affine nz64 family at --nf 48 (F = [48, 48, 96, 96, 192, 192, 384, 384]), nz_cond 20,
    nz_cond2 7 (27 condition channels) and reduce_dim 6: convolutions whose widths are not multiples of 32, an odd
    condition width, a 6-wide bottleneck;
  * `default_nf32`: the reference's default model (configs/default_config.yaml: residual encoder, conditioned encoder,
    GroupNorm decoder, reduce_dim 4) at --nf 32: the last GroupNorm blocks are 16 channels wide.

    python tests/golden/make_ref_golden_widths.py          (about a minute)
"""
import os

import numpy as np

import make_ref_golden as G
import make_ref_golden_resblock as G3

OUT = os.path.join(G.HERE, "ref_models_golden_4.npz")


def widths(nf):
    """F of the 8-layer model at --nf (config_parser.model_params)."""
    return [nf, nf, 2 * nf, 2 * nf, 4 * nf, 4 * nf, 8 * nf, 8 * nf]


def configs():
    from cape_b200.params import DEFAULTS, NZ64_AFFINE
    return (("affine_nf48", dict(NZ64_AFFINE, F=widths(48), nz_cond=20, nz_cond2=7, reduce_dim=6, decay_steps=10),
             2, 100),
            ("default_nf32", dict(DEFAULTS, F=widths(32), reduce_dim=4, affine=False, lambda_edge=0.0, decay_steps=10,
                                  use_res_block=True, cond_encoder=True), 2, 100))


def load():
    with np.load(OUT) as f:
        return {k: f[k] for k in f.files}


def main():
    from cape_b200 import topology as T
    L, D, U, p, L_d, D_d, _ = T.load_graph_mtx(load_for_demo=True)
    h = dict(L=L, D=D, U=U, p=p, L_d=L_d, D_d=D_d)
    store = {}
    for tag, cfg, N, step in configs():
        params, batch = G.inputs(cfg, h, N)
        res = G.run_reference(cfg, h, params, batch, step)
        print("%s: x_hat %s  recon %.6f edge %.6f latent %.6f gan_g %.6f gan_d %.6f  lr %s  (%d variables)"
              % (tag, res["x_hat"].shape, res["recon"], res["edge"], res["latent"], res["gan_g"], res["gan_d"], res["lr"],
                 len(res["created"])))
        G.pack(tag, res, store)
        for k in [k for k in store if k.startswith(tag + "/") and k.endswith("#full") and store[k].size > G3.FULL_MAX]:
            v = store.pop(k).reshape(-1)
            store[k[:-len("#full")] + "#sample"] = v[G.sample_index(k.split("/", 2)[2][:-len("#full")], v.size)]
    np.savez_compressed(OUT, **store)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
