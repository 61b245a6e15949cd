#!/usr/bin/env python
"""Golden vectors of the reference's DEFAULT encoder: residual encoder blocks and the conditioned encoder.
Runs only where $CAPE_REFERENCE names a checkout.

The reference's unmodified `lib/models.py` runs on the TensorFlow-1 API shim exactly as in make_ref_golden.py (same
inputs, same packing) for two cases, written to tests/golden/ref_models_golden_3.npz:

  * `default`: configs/default_config.yaml -- DEFAULTS + use_res_block 1, cond_encoder 1, reduce_dim 4, affine 0
    (the GroupNorm decoder), lambda_edge 0 -- at batch 1: one training update as `pack()` stores it, plus the
    demo-phase graph (`op_vae_mean` / `op_vae_var`, which see the condition embeddings, and `op_decoder`);
  * `res_affine`: the benchmarked affine-decoder nz64 family with the same encoder, at batch 2: one training update.

    python tests/golden/make_ref_golden_resblock.py          (about a minute)
"""
import os

import numpy as np

import make_ref_golden as G

OUT = os.path.join(G.HERE, "ref_models_golden_3.npz")
FULL_MAX = 1024         # tensors up to this size are stored in full, larger ones as G.NSAMPLE samples: keeps the file < 1 MB


def configs():
    from cape_b200.params import DEFAULTS, NZ64_AFFINE
    res = dict(use_res_block=True, cond_encoder=True)
    return (("default", dict(DEFAULTS, reduce_dim=4, affine=False, lambda_edge=0.0, decay_steps=10, **res), 1, 100),
            ("res_affine", dict(NZ64_AFFINE, decay_steps=10, **res), 2, 100))


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
        for k in [k for k in store if k.startswith(tag + "/") and k.endswith("#full") and store[k].size > FULL_MAX]:
            v = store.pop(k).reshape(-1)
            store[k[:-len("#full")] + "#sample"] = v[G.sample_index(k.split("/", 2)[2][:-len("#full")], v.size)]
        if tag == "default":
            for k, v in G.run_reference_demo(cfg, h, params, batch).items():
                store["%s/demo/%s" % (tag, k)] = v
    np.savez_compressed(OUT, **store)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
