#!/usr/bin/env python
"""The variables the reference histograms (`tf.summary.histogram(var.op.name, var)` in `_weight_variable` /
`_bias_variable`, lib/models.py:217-227), recorded from its own `build_graph(phase='train')`.  Runs only where
$CAPE_REFERENCE names a checkout.

The reference's unmodified `lib/models.py` runs on the TensorFlow-1 API shim (oracle/tf1_shim.py) as in
make_ref_golden.py, with `tf.summary.histogram` replaced for the duration of the build by a recorder, for four models:
affine nz64, GroupNorm nz18, the default model (residual and conditioned encoder) and the plain decoder.  The names are
written to tests/golden/histogram_inventory.json.

    python tests/golden/make_histogram_inventory.py
"""
import contextlib
import io
import json
import os

import make_ref_golden as G

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "histogram_inventory.json")


def configs():
    from cape_b200.params import DEFAULTS, NZ18_PLAIN, NZ64_AFFINE
    return (("affine_nz64", dict(NZ64_AFFINE, decay_steps=10)), ("groupnorm_nz18", dict(NZ18_PLAIN, decay_steps=10)),
            ("default", dict(DEFAULTS, reduce_dim=4, use_res_block=True, cond_encoder=True, decay_steps=10)),
            ("plain_decoder", dict(DEFAULTS, use_res_block_dec=False, decay_steps=10)))


def reference_histograms(cfg, h, N=1):
    """var.op.name of every tf.summary.histogram call of the reference's build_graph(phase='train'), in call order."""
    from oracle import tf1_shim as S
    from cape_b200 import topology as T
    S.install(template_vertices=T.template_mesh()[0])
    params, batch = G.inputs(cfg, h, N)
    feeds = dict(data_g=batch["x_g"], data_d=batch["x_d"], condition_g=batch["cond_g"], condition2_g=batch["cond2_g"],
                 condition_d=batch["cond_d"], condition2_d=batch["cond2_d"], gt=batch["gt"], eps=batch["eps"])
    S.reset(feeds=feeds, params=params, global_step=100)
    names = []
    saved = S.tf.summary.histogram
    S.tf.summary.histogram = lambda name, values, *a, **k: names.append(name)
    try:
        with contextlib.redirect_stdout(io.StringIO()):
            from lib import models as RM
            model = RM.CAPE(**G.reference_kwargs(cfg, h, N))
            model.build_graph(model.input_num_verts, model.nn_input_channel, phase="train")
    finally:
        S.tf.summary.histogram = saved
    return names


def main():
    from cape_b200 import topology as T
    L, D, U, p, L_d, D_d, _ = T.load_graph_mtx(load_for_demo=True)
    h = dict(L=L, D=D, U=U, p=p, L_d=L_d, D_d=D_d)
    out = {tag: reference_histograms(cfg, h) for tag, cfg in configs()}
    with open(OUT, "w") as f:
        json.dump(out, f, indent=1)
        f.write("\n")
    for tag, names in out.items():
        print(tag, len(names), "histograms,", len(set(names)), "distinct names")


if __name__ == "__main__":
    main()
