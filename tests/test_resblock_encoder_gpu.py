"""The reference's default encoder on the GPU: the pass-through term of cape_cheb_fwd through the C ABI against float64,
and the residual / conditioned encoder of CapeNetwork against the oracle (tests/resblock_oracle.py) and against the
reference's own numbers (tests/golden/ref_models_golden_3.npz).

The file name sorts after every existing GPU test file, so that in one `pytest -m gpu` process the existing tests run
after exactly the tests they ran after before, in the same process state.  The kernel-selection checks here and in
tests/test_gpu_thin_paths.py rely on torch.profiler's CUDA activity records, and the profiler now and then returns a
session without any device records at all (the same happens with the library without this file's kernels, in the
same test order); running this file's work in front of those checks made three such losses on one case more likely."""
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))

import make_ref_golden as G  # noqa: E402
import make_ref_golden_resblock as G3  # noqa: E402
import parity  # noqa: E402
import resblock_oracle as R  # noqa: E402
import test_gpu_thin_paths as TP  # noqa: E402

pytestmark = pytest.mark.gpu


def _cfg(tag):
    return next(c for t, c, n, s in G3.configs() if t == tag)


# ---- the pass-through term through the C ABI ----------------------------------------------------------------------
def _ops(hierarchy):
    """identity on level 1, the pooling D_1 (level 1 -> 2, one tap per row) and its transpose (at most one tap)."""
    D = sp.csr_matrix(hierarchy["D"][1]).astype(np.float32)
    p1 = hierarchy["L"][1].shape[0]
    return {"I": (None, p1, p1), "D": (D, D.shape[0], D.shape[1]), "DT": (sp.csr_matrix(D.T), D.shape[1], D.shape[0])}


@pytest.mark.parametrize("tc", [True, False])
@pytest.mark.parametrize("epi", ["linear", "slope"])
@pytest.mark.parametrize("opk", ["I", "D", "DT"])
@pytest.mark.parametrize("ncols", [64, 128, 256, 512])
def test_pass_through_term(hierarchy, ncols, opk, epi, tc):
    """out = epi(op x W + op s + bias), pass-through term op s (F == ncols) mixed with a contracted term of the same
    operator; NaN-filled guarded output, the kernel that ran checked by tracing."""
    E = TP._E()
    tp = TP._tp()
    m, rows_out, rows_in = _ops(hierarchy)[opk]
    op = -1 if m is None else tp.add_operator(m)
    rng = np.random.RandomState(ncols + len(opk) + (7 if tc else 0))
    N, F = 2, 64
    x = rng.randn(N, rows_in, F).astype(np.float32)
    s = rng.randn(N, rows_in, ncols + 4).astype(np.float32)        # src_stride > F: columns past F are NaN
    s[:, :, ncols:] = np.nan
    W = (rng.randn(F, ncols) * 0.1).astype(np.float32)
    b = (rng.randn(ncols) * 0.1).astype(np.float32)
    aux = rng.randn(N, rows_out, ncols).astype(np.float32)
    dev = TP._dev()
    xd, sd, Wd = torch.from_numpy(x).to(dev), torch.from_numpy(s).to(dev), torch.from_numpy(W).to(dev)
    WTd = Wd.t().contiguous()
    bd, auxd = torch.from_numpy(b).to(dev), torch.from_numpy(aux).to(dev)
    total = N * rows_out * ncols
    init = np.full(total + TP.GUARD, np.nan, np.float32)
    init[total:] = 7.0
    outd = torch.from_numpy(init).to(dev)
    terms = [dict(src=xd, op=op, F=F, src_rows=rows_in, src_stride=F, w=Wd, w_stride=ncols, wT=WTd, wT_stride=F),
             dict(src=sd, op=op, F=ncols, src_rows=rows_in, src_stride=ncols + 4, w=None, w_stride=0)]
    kw = dict(bias=bd, act=E.ACT_LEAKY) if epi == "linear" else dict(epilogue=E.EPI_SLOPE, aux=auxd)

    def call():
        E.cheb_call(tp, N, rows_out, ncols, terms, outd, **kw)

    def reset():
        outd.copy_(torch.from_numpy(init))

    with TP._knobs(tc=tc):
        names = TP._traced(call, reset)
    TP._expect(names, ["conv_wg_kernel" if tc else "ellconv_kernel"], launches=1, thin=False)
    acc = TP._apply(m, x) @ W.astype(np.float64) + TP._apply(m, s[:, :, :ncols])
    if epi == "linear":
        acc = acc + b
        want = np.where(acc > 0, acc, 0.2 * acc)
    else:
        want = acc * np.where(aux > 0, 1.0, 0.2)
    want_all = np.concatenate([want.reshape(-1), np.full(TP.GUARD, 7.0)])
    mask = np.zeros(total + TP.GUARD, bool)
    mask[:total] = True
    err = TP._check(outd.cpu().numpy(), init, mask, want_all, "pass-through %s %d %s tc=%s" % (opk, ncols, epi, tc))
    TP._report("pass-through %s ncols=%d %s tc=%d" % (opk, ncols, epi, tc), err)


def test_invalid_pass_through_calls_are_refused(hierarchy):
    from cape_b200 import _lib
    E = TP._E()
    tp = TP._tp()
    dev = TP._dev()
    rows, F, nc = hierarchy["L"][1].shape[0], 64, 64
    x = torch.randn(1, rows, F, device=dev)
    W = torch.randn(F, nc, device=dev)
    WT = W.t().contiguous()
    out = torch.zeros(1, rows, nc, device=dev)
    y = torch.randn(1, 8, device=dev)
    conv = dict(src=x, op=-1, F=F, src_rows=rows, src_stride=F, w=W, w_stride=nc, wT=WT, wT_stride=F)
    pas = dict(src=x, op=-1, F=nc, src_rows=rows, src_stride=F, w=None, w_stride=0)
    bad = [([conv, dict(pas, F=32)], {}),                                   # F != ncols
           ([conv, dict(pas, wc=W[:8])], dict(cond=y)),                     # condition rows
           ([conv, dict(pas, stash=out, stash_stride=nc)], {}),             # a basis copy
           ([pas], {}),                                                     # nothing contracted
           ([dict(conv, w=None), pas], dict(plain_only=True))]              # plain_only
    for terms, kw in bad:
        with pytest.raises(_lib.CapeError):
            E.cheb_call(tp, 1, rows, nc, terms, out, **kw)
    torch.cuda.synchronize()


# ---- the network ------------------------------------------------------------------------------------------------------
def _assert_parity(res, what):
    bad = {k: v for k, v in res.items() if not k.startswith("unmasked") and not v < parity.TOL}
    assert not bad, (what, bad)
    unm = {k: v for k, v in res.items() if k.startswith("unmasked") and "max-rel" not in k and not v < parity.TOL}
    assert not unm, (what, unm)


@pytest.mark.parametrize("mode", ["eager", "graph", "reorder"])
def test_default_model_update_matches_oracle(hierarchy, mode):
    res = R.train_step(hierarchy, _cfg("default"), N=2, use_graph=mode == "graph", reorder=mode == "reorder")
    print("default %s: worst %s" % (mode, max(res.items(), key=lambda kv: kv[1])))
    _assert_parity(res, mode)


def test_res_affine_model_update_at_batch_64_matches_oracle(hierarchy):
    """The benchmarked model family with the new encoder at batch 64, through the captured graphs.  The residual
    encoder's outputs are larger than the plain one's, so the fc kernels are scaled down further than parity's default
    (0.05): at 0.05 the log-variances reach the range where exp() in the KL term turns fp32 rounding of the encoder
    output into 1e-4 of the KL loss and of every gradient that flows through it, in any fp32 implementation."""
    res = R.train_step(hierarchy, _cfg("res_affine"), N=64, use_graph=True, fc_scale=0.01)
    print("res_affine N=64: worst %s" % (max(res.items(), key=lambda kv: kv[1]),))
    _assert_parity(res, "res_affine N=64")


@pytest.mark.parametrize("tag", ["default", "res_affine"])
def test_update_matches_the_reference_golden(hierarchy, tag):
    """The update ref_models_golden_3.npz holds, on the CUDA path: x_hat, the losses and the discriminator's post-update
    parameters (what parity.reference_golden_update compares for the shipped models, for the same reasons)."""
    from cape_b200.network import CapeNetwork
    cfg, N, step = next((c, n, s) for t, c, n, s in G3.configs() if t == tag)
    h = hierarchy
    params, batch = G.inputs(cfg, h, N)
    net = CapeNetwork(h["L"], h["D"], h["U"], h["L_d"], h["D_d"], cfg, N, params=params, ref_compat=True)
    tb = {k: torch.from_numpy(v) for k, v in batch.items()}
    net.set_inputs(tb["x_g"], tb["cond_g"], tb["cond2_g"], tb["eps"], tb["x_d"], tb["cond_d"], tb["cond2_d"])
    net.train_step(step=step)
    torch.cuda.synchronize()
    z = G3.load()
    out = {"x_hat (vertex-L2)": parity.vertex_l2(net.x_hat.cpu().numpy(), z[tag + "/x_hat"])}
    got = net.loss_dict()
    for k in ("recon", "edge", "latent", "gan_g", "gan_d"):
        want = float(z["%s/%s" % (tag, k)])
        out["loss " + k] = abs(got[k] - want) / max(abs(want), 1e-30)
    for name, v in net.get_params().items():
        if name.startswith("discriminator"):
            base = "%s/params_after/%s" % (tag, name)
            v = v.reshape(-1)
            ref = z[base + "#full"] if base + "#full" in z else z[base + "#sample"]
            out["param " + name] = parity.rel(v if base + "#full" in z else v[G.sample_index(name, v.size)],
                                              ref.reshape(-1))
    print("%s vs reference: worst %s" % (tag, max(out.items(), key=lambda kv: kv[1])))
    assert max(out.values()) < parity.TOL, {k: v for k, v in out.items() if not v < parity.TOL}


def test_encode_decode_predict_with_the_conditioned_encoder(hierarchy):
    from cape_b200.models import CAPE
    from cape_b200.synthetic import make_batch
    h = hierarchy
    cfg = _cfg("default")
    kw = G.reference_kwargs(cfg, dict(h, p=h["p"]), 4)
    m = CAPE(**kw)
    m.build_graph(m.input_num_verts, m.nn_input_channel, phase="demo")
    params = parity.calibrated_params(m.net.specs, 11)
    m.load_weights(params)
    n = 6
    b = make_batch(n, cfg["nz"], seed=5)
    o = R.ResOracle(h["L"], h["D"], h["U"], h["L_d"], h["D_d"], cfg)
    P = {k: torch.from_numpy(v) for k, v in params.items()}
    t = torch.from_numpy
    with torch.no_grad():
        y, y2 = o.cond_embeddings(t(b["cond_g"]), t(b["cond2_g"]), P)
        zm, zl = o.encoder(t(b["x_g"]), P, y, y2)
    gm, gl, gc, gc2 = m.encode(b["x_g"], b["cond_g"], b["cond2_g"])
    assert parity.rel(gm, zm.numpy()) < parity.TOL and parity.rel(gl, zl.numpy()) < parity.TOL
    z = np.random.RandomState(0).normal(size=(n, cfg["nz"])).astype(np.float32)
    z_total = np.concatenate([z, gc, gc2], 1)
    with torch.no_grad():
        want = o.decoder_cond_vert(t(z_total), y, y2, P).numpy()
    assert parity.vertex_l2(m.decode(z_total, gc, gc2), want) < parity.TOL
    m.rng = np.random.RandomState(123)
    rng = np.random.RandomState(123)
    eps = np.concatenate([rng.normal(size=(4, cfg["nz"])), rng.normal(size=(4, cfg["nz"]))]).astype(np.float32)
    preds = m.predict(b["x_g"], b["cond_g"], b["cond2_g"])
    xw = []
    with torch.no_grad():
        for s in (slice(0, 4), slice(4, 6)):
            xh, _, _ = o.generator(t(b["x_g"][s]), y[s], y2[s], t(eps[s]), P)
            xw.append(xh.numpy())
    assert parity.vertex_l2(preds, np.concatenate(xw)) < parity.TOL


def test_tensorflow_checkpoint_of_the_default_model_restores_by_name(hierarchy, tmp_path):
    from cape_b200 import tf_checkpoint
    from cape_b200.network import CapeNetwork
    h = hierarchy
    cfg = _cfg("default")
    net = CapeNetwork(h["L"], h["D"], h["U"], h["L_d"], h["D_d"], cfg, 1)
    params = parity.calibrated_params(net.specs, 3)
    prefix = str(tmp_path / "model.ckpt-5")
    tf_checkpoint.write_checkpoint(prefix, dict(params, global_step=np.asarray(5, np.int64)))
    names = {n for n, _, _ in tf_checkpoint.list_variables(prefix)}
    assert {n for n in names if "encoder_resblock" in n} == {n for n in net.specs if "encoder_resblock" in n}
    net.set_params(tf_checkpoint.read_checkpoint(prefix, names=list(net.specs)))
    got = net.get_params()
    assert all(np.array_equal(got[k], params[k]) for k in params)


def test_no_encoder_conv2_launch_runs_on_the_fp32_kernel(hierarchy):
    """With tensor cores on, every block's fused conv2 + skip launch (forward) and conv1 + skip launch (data gradient)
    takes the wgmma kernel: the first block's 3-channel projection runs on the thin kernel and enters as a
    pass-through term, so no launch of a block falls back to ellconv_kernel."""
    from cape_b200.network import CapeNetwork
    from cape_b200.synthetic import make_batch
    h = hierarchy
    cfg = _cfg("default")
    N = 2
    net = CapeNetwork(h["L"], h["D"], h["U"], h["L_d"], h["D_d"], cfg, N)
    tb = {k: torch.from_numpy(v) for k, v in make_batch(N, cfg["nz"], seed=1).items()}
    net.set_inputs(tb["x_g"], tb["cond_g"], tb["cond2_g"], tb["eps"], tb["x_d"], tb["cond_d"], tb["cond2_d"])
    with TP._knobs(tc=True):
        net.train_step(update=False)
        torch.cuda.synchronize()
        for b in net.enc:
            x = net.enc_act[b.i - 1] if b.i else net.in_x
            yc = net.ycat_g if b.i == 0 else None
            names = TP._traced(lambda: b.fwd(x, yc, net.enc_act[b.i]), lambda: None)
            assert names[-1].startswith("conv_wg_kernel"), (b.i, names)          # conv2 + skip is the last launch
            assert not TP._ran(names, "ellconv_kernel"), (b.i, names)
            if b.i:
                bwd = lambda: b.bwd(x, None, net.g_enc[b.i], dx=net.g_enc[b.i - 1], dx_aux=x)
            else:
                bwd = lambda: b.bwd(x, yc, net.g_enc[0], dycat=net.d_ycat)
            names = TP._traced(lambda: (bwd(), net.join_dw()), lambda: None)
            assert not TP._ran(names, "ellconv_kernel"), (b.i, names)
            if b.i:
                assert TP._ran(names, "conv_wg_kernel"), (b.i, names)
        net.small.flush()
        torch.cuda.synchronize()
