"""The network at layer widths the shipped configurations never use, and the fp32 gather kernels those widths select.

At the shipped widths every wide conv is a multiple of 32 columns, so with tensor cores on the wgmma and thin kernels
take every launch and the fp32 kernels of csrc/ellconv.cu (ellconv_kernel, ellconv_dw_kernel + reduce_splits_kernel, the
forward's basis copies by resample_kernel) never run in a training step.  --nf, --nz_cond, --nz_cond2 and reduce_dim
reach them:

- network cases, against the oracle and against the reference's own numbers (tests/golden/ref_models_golden_4.npz):
  `affine_nf48` (the affine nz64 family at --nf 48, 27 condition channels, reduce_dim 6) and `default_nf32` (the
  reference's default model at --nf 32: 16-channel GroupNorm blocks), with a census of the kernels their odd layers
  launch, so that the network cases cannot pass without running the fp32 kernels;
- kernel cases through cape_cheb_fwd / cape_cheb_dw against a float64 NumPy / SciPy product at the shapes where the fp32
  kernels branch: scalar and float4 columns, partial column tiles, F not a multiple of 4, several terms, two
  accumulators, condition slots over tiles that span many samples, every epilogue, basis copies, split-K and direct
  stores.  Every case checks which kernels ran, that every element it should write is finite and within 1e-4 of
  max |truth|, and that sentinels after its outputs, in the columns past F of a basis copy and in neighbouring
  weight-gradient slices are untouched.

The file name sorts after every other GPU test file (see tests/test_resblock_encoder_gpu.py for why that matters)."""
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))

import make_ref_golden_widths as G4  # noqa: E402
import parity  # noqa: E402
import resblock_oracle as R  # noqa: E402
import test_gpu_thin_paths as TP  # noqa: E402
import test_resblock_encoder_gpu as RG  # noqa: E402

pytestmark = pytest.mark.gpu

NAN = TP.NAN
C27 = 27                 # nz_cond 20 + nz_cond2 7 of affine_nf48


def _cfg(tag):
    return next(c for t, c, n, s in G4.configs() if t == tag)


def _count(names, kernel):
    return sum(TP._ran([n], kernel) for n in names)


def _fp32_conv(ncols, dual):
    return "ellconv_kernel<%d, %s, false>" % (32 if ncols <= 32 else 64, "true" if dual else "false")


# =====================================================================================================================
# the network
# =====================================================================================================================
def _assert_all(res, what):
    bad = {k: v for k, v in res.items() if not v < parity.TOL}
    print("%s: %d values, worst %s" % (what, len(res), max(res.items(), key=lambda kv: kv[1])))
    assert not bad, (what, bad)


@pytest.mark.parametrize("mode", ["eager", "graph"])
def test_affine_nf48_update_matches_oracle(hierarchy, mode):
    """Batch 2 eager, batch 5 replayed from the captured graphs; every gradient, clipped update and parameter."""
    res = parity.train_step(hierarchy, _cfg("affine_nf48"), N=2 if mode == "eager" else 5, use_graph=mode == "graph")
    _assert_all(res, "affine_nf48 " + mode)


def test_affine_nf48_vs_float64_truth(hierarchy):
    """The reference's initialisers (fc_scale 1: logvar up to +-10): within 1e-4 of the float64 oracle, or at least as
    close as twice what the fp32 oracle gets on the same update."""
    res = parity.train_step(hierarchy, _cfg("affine_nf48"), N=2, fc_scale=1.0, truth=True)
    print("affine_nf48 vs fp64: worst %s" % (max(res.items(), key=lambda kv: kv[1][0]),))
    bad = {k: v for k, v in res.items() if not v[0] < max(parity.TOL, 2.0 * v[1])}
    assert not bad, "further from the fp64 truth than an fp32 CPU implementation (err, fp32-oracle err): %s" % bad


@pytest.mark.parametrize("mode", ["eager", "graph"])
def test_default_nf32_update_matches_oracle(hierarchy, mode):
    """Tensor cores off: every conv of the step on the fp32 kernels, against the fp32 oracle at 1e-4.  With tensor
    cores on (the default) the encoder's gradients do not meet that bound; test_default_nf32_vs_float64_truth says
    why and what they meet instead."""
    with TP._knobs(tc=False):
        res = R.train_step(hierarchy, _cfg("default_nf32"), N=2, use_graph=mode == "graph")
    print("default_nf32 %s tc=0: worst %s" % (mode, max(res.items(), key=lambda kv: kv[1])))
    RG._assert_parity(res, mode)


ENC_GRAD_TOL = 2e-4      # default_nf32, tensor cores on: the encoder's gradients against float64 (see below)


@pytest.mark.parametrize("tc", [True, False])
def test_default_nf32_vs_float64_truth(hierarchy, tc):
    """default_nf32 against the float64 oracle (the CUDA branch decisions imposed on it).

    Every forward activation -- the eight encoder blocks, the bottleneck, z_total, the decoder's fc and blocks, x_hat --
    has to be within 1e-5 of the truth with tensor cores on or off: that is where a defective contraction at these
    widths would show (measured on an H100: at most 4.6e-6 on, 3.1e-6 off).  Every gradient outside the encoder has to
    be within 1e-4.  The encoder's gradients amplify the forward's rounding: with tensor cores off they are 4e-6 from
    the truth, on (3xTF32 forward activations 1e-6 .. 4e-6 from the truth instead of 3e-7 .. 1.4e-6) 1.2e-4 -- at
    encoder_resblock2/bias_relu_1, 1.4e-5 when only the encoder's forward runs without tensor cores, with no single
    block carrying it.  So they are held to ENC_GRAD_TOL with tensor cores on and to 1e-4 off."""
    from oracle import cape_oracle as O
    from cape_b200 import topology as T
    from cape_b200.network import CapeNetwork
    from cape_b200.params import param_specs
    from cape_b200.synthetic import make_batch
    h, cfg, N, step, seed = hierarchy, _cfg("default_nf32"), 2, 100, 123
    params = parity.calibrated_params(param_specs(cfg, [l.shape[0] for l in h["L"]], [l.shape[0] for l in h["L_d"]]),
                                      seed, 0.05)
    tb = {k: torch.from_numpy(v) for k, v in make_batch(N, cfg["nz"], seed=seed).items()}
    with TP._knobs(tc=tc):
        net = CapeNetwork(h["L"], h["D"], h["U"], h["L_d"], h["D_d"], cfg, N, params=params)
        net.set_inputs(tb["x_g"], tb["cond_g"], tb["cond2_g"], tb["eps"], tb["x_d"], tb["cond_d"], tb["cond2_d"])
        net.train_step(step=step)
        torch.cuda.synchronize()
    got = net.get_grads()
    o = R.ResOracle(h["L"], h["D"], h["U"], h["L_d"], h["D_d"], cfg, dtype=torch.float64)
    o.masks, o.mask_rows = R.cuda_masks(net, h, N)
    o.keep = {}
    P = {k: torch.from_numpy(np.asarray(v)).double() for k, v in params.items()}
    M = {k: torch.zeros_like(v) for k, v in P.items()}
    truth = O.train_update(o, P, M, {k: v.double() for k, v in tb.items()}, step, T.smpl_edges())
    fwd = {"x_hat": parity.rel(net.x_hat.cpu().numpy(), truth["x_hat"].numpy())}
    mine = dict([("enc_act%d" % (i + 1), a) for i, a in enumerate(net.enc_act)] +
                [("dec_act%d" % (i + 1), a) for i, a in enumerate(net.dec_act)] +
                [("enc_red", net.enc_red), ("z_total", net.z_total), ("dec_fc", net.dec_fc)])
    for k, a in mine.items():
        fwd[k] = parity.rel(a.cpu().numpy(), o.keep[k].detach().numpy())
    grads = {k: parity.rel(got[k].reshape(-1), g.numpy().reshape(-1)) for k, g in truth["grads"].items()}
    print("default_nf32 tc=%d vs fp64: forward worst %s, gradient worst %s" % (
        tc, max(fwd.items(), key=lambda kv: kv[1]), max(grads.items(), key=lambda kv: kv[1])))
    assert len(fwd) == 20 and max(fwd.values()) < 1e-5, fwd
    enc_tol = ENC_GRAD_TOL if tc else parity.TOL
    bad = {k: v for k, v in grads.items() if not v < (enc_tol if k.startswith("generator/encoder/") else parity.TOL)}
    assert not bad, bad


@pytest.mark.parametrize("tag", ["affine_nf48", "default_nf32"])
def test_update_matches_the_reference_golden(hierarchy, tag):
    """The update ref_models_golden_4.npz holds, on the CUDA path."""
    out = RG.golden_update_errors(hierarchy, G4.configs, G4.load, tag)
    assert max(out.values()) < parity.TOL, {k: v for k, v in out.items() if not v < parity.TOL}


# ---- kernel census ---------------------------------------------------------------------------------------------------
def _net(hierarchy, tag, N=2):
    from cape_b200.network import CapeNetwork
    from cape_b200.synthetic import make_batch
    h = hierarchy
    cfg = _cfg(tag)
    net = CapeNetwork(h["L"], h["D"], h["U"], h["L_d"], h["D_d"], cfg, N)
    tb = {k: torch.from_numpy(v) for k, v in make_batch(N, cfg["nz"], seed=1).items()}
    net.set_inputs(tb["x_g"], tb["cond_g"], tb["cond2_g"], tb["eps"], tb["x_d"], tb["cond_d"], tb["cond2_d"])
    return net


def _census(net, label, fn, must, absent=()):
    """Traces one layer call (and the weight gradients it leaves on the side stream); every kernel in `must` has to be
    among the launches, none of `absent`."""
    names = TP._traced(lambda: (fn(), net.join_dw()), lambda: None)
    print("census %-40s %s" % (label, names))
    for k in must:
        assert TP._ran(names, k), "%s: expected %s, launched %s" % (label, k, names)
    for k in absent:
        assert not TP._ran(names, k), "%s: %s ran: %s" % (label, k, names)
    return names


def test_census_affine_nf48(hierarchy):
    """Which kernels the layers of affine_nf48 that leave the 32-column grid launch, tensor cores on."""
    net = _net(hierarchy, "affine_nf48")
    TC = ("conv_wg_kernel", "dw_wg_kernel")
    with TP._knobs(tc=True):
        net.train_step(update=False)
        torch.cuda.synchronize()
        e, d, yc = net.enc, net.dec, net.ycat_g
        slope = lambda i: dict(dx=net.g_enc[i - 1], dx_epi=TP._E().EPI_SLOPE, dx_aux=net.enc_act[i - 1])
        # enc/conv1 (3 -> 48): thin forward; dW with F = 3 and 48 columns is not a thin_dw shape
        _census(net, "enc/conv1 fwd", lambda: e[0].fwd(net.in_x, None, net.enc_act[0]), ["thin_fwd_kernel"])
        names = _census(net, "enc/conv1 bwd", lambda: e[0].bwd(net.in_x, None, net.g_enc[0]), ["ellconv_dw_kernel"],
                        ("thin_dw_kernel",) + TC)
        assert _count(names, "ellconv_dw_kernel") == 2
        # enc/conv2 (48 -> 48, pooled): forward and data gradient fused on the fp32 kernel, dW gathered again
        assert e[1].dw_mode == "gather" and (e[1].fwd_mode, e[1].dx_mode) == ("fused", "fused")
        _census(net, "enc/conv2 fwd", lambda: e[1].fwd(net.enc_act[0], None, net.enc_act[1]),
                [_fp32_conv(48, False)], TC)
        names = _census(net, "enc/conv2 bwd", lambda: e[1].bwd(net.enc_act[0], None, net.g_enc[1], **slope(1)),
                        [_fp32_conv(48, False), "ellconv_dw_kernel"], TC)
        assert _count(names, "ellconv_dw_kernel") == 2
        # enc/conv3 (48 -> 96): the gradient narrows, so its 48-column data gradient is contract-first (a tensor-core
        # projection to K * 48 = 96 columns, then the operators by cape_apply), not a fused fp32 launch
        assert (e[2].dw_mode, e[2].dx_mode) == ("aside", "contract")
        _census(net, "enc/conv3 bwd", lambda: e[2].bwd(net.enc_act[1], None, net.g_enc[2], **slope(2)),
                ["conv_wg_kernel", "apply_kernel"], ("ellconv_kernel",))
        # enc/1x1 (384 -> 6) and dec/1x1 (6 -> 384): 6 columns / F = 6
        _census(net, "enc/1x1 fwd", lambda: net.enc_1x1.fwd(net.enc_act[-1], None, net.enc_red), [_fp32_conv(6, False)],
                TC)
        _census(net, "enc/1x1 bwd", lambda: net.enc_1x1.bwd(net.enc_act[-1], None, net.g_enc_red, dx=net.g_enc[-1],
                                                            dx_epi=TP._E().EPI_SLOPE, dx_aux=net.enc_act[-1]),
                [_fp32_conv(384, False), "ellconv_dw_kernel"], TC)
        fcv = net.dec_fc.view(net.N, net.p[-1], net.red)
        _census(net, "dec/1x1 fwd", lambda: net.dec_1x1.fwd(fcv, None, net.dec_h0), [_fp32_conv(384, False)], TC)
        _census(net, "dec/1x1 bwd", lambda: net.dec_1x1.bwd(fcv, None, net.g_dec_h0,
                                                            dx=net.g_dec_fc.view(net.N, net.p[-1], net.red)),
                [_fp32_conv(6, False), "ellconv_dw_kernel"], TC)
        # dec/aff7 (48 -> 24) and dec/aff8 (24 -> 24): fused, two accumulators, 27 condition channels
        for i in (6, 7):
            lay = d[i]
            assert lay.Fout == 24 and lay.C == C27 and (lay.fwd_mode, lay.dx_mode) == ("fused", "fused")
            _census(net, "%s fwd" % lay.name, lambda: lay.fwd(net.dec_act[i - 1], yc, net.dec_act[i], out2=net.dec_rg[i]),
                    [_fp32_conv(24, True)], TC)
            names = _census(net, "%s bwd" % lay.name,
                            lambda: lay.bwd(net.dec_act[i - 1], yc, net.g_dec_m[i], g_aff=net.g_dec[i],
                                            dx=net.g_dec[i - 1], dx2=net.g_dec_m[i - 1], dx_epi=TP._E().EPI_DUALMASK,
                                            dx_aux=net.dec_rg[i - 1], dycat=net.d_ycat),
                            [_fp32_conv(lay.F, False), "ellconv_dw_kernel", "colsum_kernel"], TC)
            assert _count(names, "ellconv_dw_kernel") == 3                     # K = 2 orders + the affine branch
        # dec/outputs (24 + 27 -> 3, per-row bias): thin-output kernels need F >= 32
        lay = net.dec_out
        _census(net, "dec/outputs fwd", lambda: lay.fwd(net.dec_act[-1], yc, net.x_hat), [_fp32_conv(3, False)],
                ("thinout_project_kernel",))
        _census(net, "dec/outputs bwd", lambda: lay.bwd(net.dec_act[-1], yc, net.d_xhat, dx=net.g_dec[-1],
                                                        dx2=net.g_dec_m[-1], dx_epi=TP._E().EPI_DUALMASK,
                                                        dx_aux=net.dec_rg[-1], dycat=net.d_ycat),
                ["ellconv_dw_kernel", "colsum_kernel"], ("thin_dw_kernel",))
        net.small.flush()
        torch.cuda.synchronize()


def test_census_default_nf32(hierarchy):
    """The last two GroupNorm blocks of default_nf32 (mid = 16): lin1, the 16 -> 16 conv and lin2 on the fp32 kernels."""
    net = _net(hierarchy, "default_nf32")
    TC = ("conv_wg_kernel", "dw_wg_kernel")
    with TP._knobs(tc=True):
        net.train_step(update=False)
        torch.cuda.synchronize()
        for i in (6, 7):
            b = net.dec[i]
            assert b.mid == 16 and b.gn[1]["G"] == 16 and b.gn[2]["G"] == 16
            _census(net, "dec/res%d lin1 fwd" % (i + 1), lambda: b.lin1.fwd(b.A1, None, b.H1), [_fp32_conv(16, False)],
                    TC)
            _census(net, "dec/res%d conv fwd" % (i + 1), lambda: b.conv.fwd(b.A2, None, b.H2), [_fp32_conv(16, False)],
                    TC)
            _census(net, "dec/res%d lin2 bwd" % (i + 1), lambda: b.lin2.bwd(b.A3, None, net.g_dec[i], dx=b.dA3),
                    [_fp32_conv(16, False), "ellconv_dw_kernel"], TC)
            names = _census(net, "dec/res%d conv bwd" % (i + 1), lambda: b.conv.bwd(b.A2, None, b.dH2, dx=b.dA2),
                            [_fp32_conv(16, False), "ellconv_dw_kernel"], TC)
            assert _count(names, "ellconv_dw_kernel") == 2
            _census(net, "dec/res%d lin1 bwd" % (i + 1), lambda: b.lin1.bwd(b.A1, None, b.dH1, dx=b.dA1),
                    [_fp32_conv(b.Ft, False), "ellconv_dw_kernel"], TC)
        net.small.flush()
        torch.cuda.synchronize()


# =====================================================================================================================
# ellconv_kernel through cape_cheb_fwd
# =====================================================================================================================
def fwd_case(N, rows_out, ncols, terms, *, C=C27, epilogue="linear", act="none", bias=None, out2=False,
             misalign=False, tp=None, seed=0):
    """terms: dicts of F, m (a scipy operator [rows_out x src_rows], or None: identity), stride (source row stride,
    default F) and the optional flags w2 (weights of the second accumulator), wc / wc2 (condition weights of
    accumulator 0 / 1) and stash (row stride of a basis copy op . src[:, :, :F]).  Weights of accumulator 0 sit at a row
    stride of 2 * ncols, those of accumulator 1 at ncols + 4, the condition rows right below them; the columns in
    between are NaN.  Every term also carries its K-major copies (wT / w2T), so that a tensor-core kernel could take
    the call wherever its shape rules allow.  misalign: out (and out2) 4 bytes off 16-byte alignment.
    Returns (kernel names, worst relative error)."""
    E, dev = TP._E(), TP._dev()
    tp = tp or TP._tp()
    rng = np.random.RandomState(seed)
    act_id, alpha = TP.ACTS[act]
    cond = rng.normal(size=(N, C)).astype(np.float32)
    acc = [np.zeros((N, rows_out, ncols)), np.zeros((N, rows_out, ncols))]
    dterms, stashes = [], []
    for spec in terms:
        F, m = spec["F"], spec.get("m")
        stride = spec.get("stride", F)
        src_rows = rows_out if m is None else m.shape[1]
        src = rng.normal(size=(N, src_rows, stride)).astype(np.float32)
        src[:, :, F:] = NAN                                     # columns past F must never be read
        basis = TP._apply(m, src[:, :, :F])
        t = dict(src=torch.from_numpy(src).to(dev), op=TP._op_id(tp, m), F=F, src_rows=src_rows, src_stride=stride)
        for a, (wk, ck, sk, tk) in enumerate((("w", "wc", "w_stride", "wT"), ("w2", "wc2", "w2_stride", "w2T"))):
            if a == 1 and not spec.get("w2"):
                continue
            ws = 2 * ncols if a == 0 else ncols + 4
            wb = np.full((F + C, ws), NAN, np.float32)
            wb[:, :ncols] = rng.normal(0, 1 / np.sqrt(F), size=(F + C, ncols))
            wd = torch.from_numpy(wb).to(dev)
            t[wk], t[sk] = wd[:F], ws
            t[tk], t[tk + "_stride"] = torch.from_numpy(np.ascontiguousarray(wb[:F, :ncols].T)).to(dev), F
            acc[a] += basis @ wb[:F, :ncols].astype(np.float64)
            if spec.get(ck):
                t[ck] = wd[F:]                                  # at the row stride of its accumulator's weights
                q = cond.astype(np.float64) @ wb[F:, :ncols].astype(np.float64)
                acc[a] += TP._rowsum(m, rows_out)[None, :, None] * q[:, None, :]
        if spec.get("stash"):
            ss = spec["stash"]
            d, init, _ = TP._buffer(N * rows_out * ss, NAN)
            mask = np.zeros(init.size, bool)
            mask[:N * rows_out * ss].reshape(N, rows_out, ss)[:, :, :F] = True
            want = np.full(init.size, np.nan)
            want[:N * rows_out * ss].reshape(N, rows_out, ss)[:, :, :F] = basis
            t["stash"], t["stash_stride"] = d, ss
            stashes.append((d, init, mask, want))
        dterms.append(t)
    total = N * rows_out * ncols
    b = None
    if bias is not None:
        b = rng.normal(size=(rows_out, ncols) if bias == "row" else (ncols,)).astype(np.float32)
    aux = rng.normal(size=(N, rows_out, ncols)).astype(np.float32) if epilogue in ("slope", "dualmask") else None
    if epilogue == "linear":
        v = acc[0] + (b.astype(np.float64) if b is not None else 0.0)
        want = [v if act == "none" else (np.maximum(v, 0) if act == "relu" else np.where(v > 0, v, alpha * v))]
    elif epilogue == "affine":
        rg = np.maximum(acc[0], 0)
        want = [acc[1] + rg] + ([rg] if out2 else [])
    elif epilogue == "slope":
        want = [acc[0] * np.where(aux > 0, 1.0, alpha)]
    else:
        want = [acc[0]] + ([np.where(aux > 0, acc[0], 0.0)] if out2 else [])
    head = 1 if misalign else 0
    outs = [TP._buffer(total, NAN, head) for _ in want]
    views = [d[head:head + total].view(N, rows_out, ncols) for d, _, _ in outs]
    epi = {"linear": E.EPI_LINEAR, "affine": E.EPI_AFFINE, "slope": E.EPI_SLOPE, "dualmask": E.EPI_DUALMASK}[epilogue]
    cond_d = torch.from_numpy(cond).to(dev) if any(s.get("wc") or s.get("wc2") for s in terms) else None
    bias_d = torch.from_numpy(b).to(dev) if b is not None else None
    aux_d = torch.from_numpy(aux).to(dev) if aux is not None else None

    def call():
        E.cheb_call(tp, N, rows_out, ncols, dterms, views[0], out2=views[1] if len(views) > 1 else None, cond=cond_d,
                    epilogue=epi, act=act_id, alpha=alpha, bias=bias_d, bias_per_row=bias == "row", aux=aux_d)

    def reset():
        for d, init, *_ in outs + stashes:
            d.copy_(torch.from_numpy(init))
    names = TP._traced(call, reset)
    err = 0.0
    for (d, init, mask), w in zip(outs, want):
        full = np.full(init.size, np.nan)
        full[head:head + total] = w.ravel()
        err = max(err, TP._check(d.cpu().numpy(), init, mask, full, "cheb_fwd out"))
    for d, init, mask, w in stashes:
        err = max(err, TP._check(d.cpu().numpy(), init, mask, w, "cheb_fwd stash"))
    return names, err


def fp32_fwd(case, *args, **kw):
    """The call runs on ellconv_kernel (tensor cores on), after one resample_kernel per basis copy."""
    names, err = fwd_case(*args, **kw)
    terms = args[3]
    nstash = sum(1 for t in terms if t.get("stash"))
    dual = any(t.get("w2") for t in terms)
    want = ["resample_kernel"] * nstash + [_fp32_conv(args[2], dual)]
    assert len(names) == len(want) and all(TP._ran([n], k) for n, k in zip(names, want)), (case, names, want)
    TP._report(case, err)


def _terms(rng, rows_out, specs):
    """specs: (F, gathered?, extra flags); gathered terms get a random operator of 1 .. 7 taps per row."""
    out = []
    for F, gathered, *flags in specs:
        d = dict(F=F, m=TP._operator(rng, rows_out, rows_out) if gathered else None)
        for f in flags:
            d.update(f)
        out.append(d)
    return out


# column widths: BN 32 (3, 6, 20, 24) and 64 (48, 100), scalar (3, 6) and float4 (20, 24, 48, 100) columns, a partial
# last column tile everywhere but 20 / 24
@pytest.mark.parametrize("ncols", [3, 6, 20, 24, 48, 100])
def test_fp32_conv_columns(ncols):
    rng = np.random.RandomState(ncols)
    terms = _terms(rng, 203, [(32, True), (32, False)])
    with TP._knobs(tc=True):
        fp32_fwd("fp32 conv ncols=%d" % ncols, 3, 203, ncols, terms, bias="shared", act="leaky", seed=ncols)


# ncols % 4 == 0 but out 4 bytes off 16-byte alignment (ovec = 0): the scalar column path; 64 columns would otherwise go
# to the tensor cores
@pytest.mark.parametrize("ncols,epilogue", [(48, "linear"), (64, "dualmask"), (24, "affine")])
def test_fp32_conv_misaligned_out(ncols, epilogue):
    rng = np.random.RandomState(ncols + 1)
    flags = {"w2": True} if epilogue == "affine" else {}
    terms = _terms(rng, 150, [(32, True, flags), (32, False)])
    with TP._knobs(tc=True):
        fp32_fwd("fp32 conv misaligned out ncols=%d %s" % (ncols, epilogue), 3, 150, ncols, terms, epilogue=epilogue,
                 bias="row" if epilogue == "linear" else None, out2=epilogue != "linear", misalign=True)


# F of 6, 13 and 27: the scalar gather, a partial reduction chunk, src_stride > F
@pytest.mark.parametrize("F", [6, 13, 27])
def test_fp32_conv_scalar_gather(F):
    rng = np.random.RandomState(F)
    terms = _terms(rng, 177, [(F, True, {"stride": F + 3}), (F, False)])
    with TP._knobs(tc=True):
        fp32_fwd("fp32 conv scalar gather F=%d" % F, 3, 177, 48, terms, bias="shared", seed=F)


# four terms of different F (40, 6, 33, 64): the chunk loop moves to the next term in the middle of the reduction,
# from a partial chunk of one term to the first chunk of the next, vec and scalar gathers alternating
@pytest.mark.parametrize("ncols", [24, 100])
def test_fp32_conv_mixed_terms(ncols):
    rng = np.random.RandomState(ncols + 2)
    terms = _terms(rng, 160, [(40, True), (6, False), (33, True, {"stride": 35}), (64, True)])
    with TP._knobs(tc=True):
        fp32_fwd("fp32 conv terms F=40,6,33,64 ncols=%d" % ncols, 3, 160, ncols, terms, act="relu", seed=3)


# K = 3 operators of the real hierarchy: pooled (discriminator level 1), un-pooled (decoder level 5) and the transposes
# of the pooled ones (the data gradient's form)
@pytest.mark.parametrize("kind", ["pool", "unpool", "transposed"])
def test_fp32_conv_hierarchy_operators(hierarchy, kind):
    from cape_b200 import engine as E
    h = hierarchy
    tp = TP._tp()
    if kind == "unpool":
        mats = E.ConvSite(tp, h["L"][5], 3, U=h["U"][5]).mats
    else:
        mats = E.ConvSite(tp, h["L_d"][1], 3, D=h["D_d"][1]).mats
        if kind == "transposed":
            mats = [sp.csr_matrix(m.T) for m in mats]
    mats = [sp.csr_matrix(m).astype(np.float32) for m in mats]
    rows_out = mats[0].shape[0]
    terms = [dict(F=24, m=m, wc=True) for m in mats]
    with TP._knobs(tc=True):
        fp32_fwd("fp32 conv K=3 %s rows %d <- %d" % (kind, rows_out, mats[0].shape[1]), 2, rows_out, 48, terms,
                 bias="shared", act="leaky")


# two accumulators: AFFINE with and without out2, a term without w2, condition weights on both accumulators; and
# ncols 288 / 512, where the wgmma kernel refuses two accumulators (2 * ncols > 512) with tensor cores on
@pytest.mark.parametrize("ncols,out2", [(24, True), (24, False), (40, True), (288, True), (512, False)])
def test_fp32_conv_dual(ncols, out2):
    rng = np.random.RandomState(ncols)
    terms = _terms(rng, 203, [(32, True, {"w2": True, "wc": True, "wc2": True}), (32, True, {"wc": True}),
                              (32, False, {"w2": True})])
    with TP._knobs(tc=True):
        fp32_fwd("fp32 conv dual affine ncols=%d out2=%d" % (ncols, out2), 3, 203, ncols, terms, epilogue="affine",
                 out2=out2)


# condition slots with C = 27 over tiles that span many samples: rows_out 1 (128 samples per tile), 5 and 203
@pytest.mark.parametrize("rows_out,N,ncols,dual", [(1, 300, 24, False), (1, 300, 6, False), (5, 60, 48, False),
                                                   (5, 60, 24, True), (203, 3, 100, True), (203, 3, 3, False)])
def test_fp32_conv_condition(rows_out, N, ncols, dual):
    rng = np.random.RandomState(rows_out + ncols)
    t0 = {"wc": True, "w2": dual, "wc2": dual}
    specs = [(32, rows_out > 1, t0), (13, False, {"wc": rows_out > 1})]
    terms = _terms(rng, rows_out, specs)
    with TP._knobs(tc=True):
        fp32_fwd("fp32 conv cond rows_out=%d N=%d ncols=%d dual=%d" % (rows_out, N, ncols, dual), N, rows_out, ncols,
                 terms, epilogue="affine" if dual else "linear", out2=dual, bias=None if dual else "shared")


# one slot of 64 columns or two of 32 at rows_out 1: 129 samples per 128-row tile do not fit the staging buffer; the
# call is refused before any launch and leaves its output alone
@pytest.mark.parametrize("ncols,dual", [(48, False), (24, True)])
def test_fp32_conv_condition_staging_refused(ncols, dual):
    from cape_b200 import _lib
    E, dev, lib = TP._E(), TP._dev(), TP._lib()
    tp = TP._tp()
    N, C, F = 200, C27, 32
    src = torch.randn(N, 1, F, device=dev)
    w = torch.randn(F + C, ncols, device=dev)
    t = dict(src=src, op=-1, F=F, src_rows=1, src_stride=F, w=w[:F], w_stride=ncols, wc=w[F:])
    if dual:
        t.update(w2=w[:F], w2_stride=ncols, wc2=w[F:])
    out = torch.full((N, 1, ncols), 7.0, device=dev)
    torch.cuda.synchronize()
    n0 = lib.cape_launch_count()
    with pytest.raises(_lib.CapeError, match="staging"):
        E.cheb_call(tp, N, 1, ncols, [t], out, cond=torch.randn(N, C, device=dev),
                    epilogue=E.EPI_AFFINE if dual else E.EPI_LINEAR)
    torch.cuda.synchronize()
    assert lib.cape_launch_count() == n0
    assert bool((out == 7.0).all())


# LINEAR with per-column / per-row bias and none / leaky / relu; SLOPE; DUALMASK with and without out2 -- float4
# (20 columns) and scalar (6) columns
@pytest.mark.parametrize("ncols", [20, 6])
@pytest.mark.parametrize("epilogue,bias,act,out2", [
    ("linear", None, "none", False), ("linear", "shared", "none", False), ("linear", "shared", "leaky.37", False),
    ("linear", "shared", "relu", False), ("linear", "row", "none", False), ("linear", "row", "leaky", False),
    ("linear", "row", "relu", False), ("slope", None, "leaky", False), ("slope", None, "leaky.37", False),
    ("dualmask", None, "none", True), ("dualmask", None, "none", False)])
def test_fp32_conv_epilogues(ncols, epilogue, bias, act, out2):
    rng = np.random.RandomState(ncols + 5)
    terms = _terms(rng, 140, [(36, True), (8, False)])
    with TP._knobs(tc=True):
        fp32_fwd("fp32 conv %s bias=%s act=%s out2=%d ncols=%d" % (epilogue, bias, act, out2, ncols), 3, 140, ncols,
                 terms, epilogue=epilogue, bias=bias, act=act, out2=out2)


# reductions under 64 (gathered) and under 32 (plain) at 64 columns: the tensor-core kernels decline them
@pytest.mark.parametrize("gathered,F", [(True, 32), (True, 60), (False, 16)])
def test_fp32_conv_short_reduction(gathered, F):
    rng = np.random.RandomState(F)
    terms = _terms(rng, 300, [(F, gathered)])
    with TP._knobs(tc=True):
        fp32_fwd("fp32 conv kred=%d gathered=%d ncols=64" % (F, gathered), 4, 300, 64, terms, bias="shared")


# basis copies on this path: resample_kernel writes op . src[:, :, :F] into rows of stash_stride > F floats (the
# columns past F are sentinels), then ellconv_kernel contracts
@pytest.mark.parametrize("ncols", [48, 24])
def test_fp32_conv_stash(ncols):
    rng = np.random.RandomState(ncols + 9)
    terms = [dict(F=24, m=TP._operator(rng, 230, 301), stash=28),
             dict(F=32, m=TP._operator(rng, 230, 301), stash=40, wc=True), dict(F=32, m=None)]
    with TP._knobs(tc=True):
        fp32_fwd("fp32 conv stash ncols=%d" % ncols, 3, 230, ncols, terms, bias="shared", act="leaky")


# =====================================================================================================================
# ellconv_dw_kernel (+ reduce_splits_kernel) through cape_cheb_dw
# =====================================================================================================================
def fp32_dw(case, N, rows_out, ncols, F, ms, *, split, **kw):
    """TP.dw_case: dW into terms 1 .. nops of a [F, nops + 2, ncols + 4] buffer (neighbouring terms and the four columns
    after every row are sentinels).  split: partials through the workspace and reduce_splits_kernel, else one split
    storing (or accumulating) directly."""
    with TP._knobs(tc=True):
        names, err = TP.dw_case(N, rows_out, ncols, F, ms, **kw)
    nops = len(ms)
    assert all(TP._ran([n], "ellconv_dw_kernel") or TP._ran([n], "reduce_splits_kernel") for n in names), (case, names)
    assert _count(names, "ellconv_dw_kernel") == nops, (case, names)
    assert _count(names, "reduce_splits_kernel") == (nops if split else 0), (case, names)
    TP._report(case, err)


# F x ncols of 3, 6, 24, 48, 100: scalar and float4 operands, partial 64 x 64 tiles, two tiles each way at 100
@pytest.mark.parametrize("ncols", [3, 6, 24, 48, 100])
@pytest.mark.parametrize("F", [3, 6, 24, 48, 100])
def test_fp32_dw_shapes(F, ncols):
    rng = np.random.RandomState(F * 7 + ncols)
    fp32_dw("fp32 dW F=%d ncols=%d" % (F, ncols), 3, 700, ncols, F, [TP._operator(rng, 700, 700)], single=True,
            split=True, seed=F + ncols)


# shapes the wgmma weight-gradient kernel takes from 4096 rows on, at 4095 / 4000 / 1000 rows; gathered and plain
@pytest.mark.parametrize("gathered", [True, False])
@pytest.mark.parametrize("F,ncols,N,rows", [(64, 64, 3, 1365), (48, 96, 2, 2000), (32, 512, 1, 1000)])
def test_fp32_dw_below_wgmma_rows(F, ncols, N, rows, gathered):
    rng = np.random.RandomState(F + ncols)
    m = TP._operator(rng, rows, rows) if gathered else None
    fp32_dw("fp32 dW below 4096 rows F=%d ncols=%d gathered=%d" % (F, ncols, gathered), N, rows, ncols, F, [m],
            single=True, split=True)


# source row strides that are not multiples of 4 (scalar gather although F % 4 == 0), plain and gathered, pooled
@pytest.mark.parametrize("gathered", [True, False])
@pytest.mark.parametrize("F,stride", [(48, 49), (24, 27), (100, 103)])
def test_fp32_dw_odd_stride(F, stride, gathered):
    rng = np.random.RandomState(stride)
    m = TP._operator(rng, 400, 650) if gathered else None
    fp32_dw("fp32 dW F=%d src_stride=%d gathered=%d" % (F, stride, gathered), 3, 400, 64, F, [m], single=True,
            split=True, src_rows=650 if gathered else 400, src_stride=stride, accumulate=True)


# split-K through the workspace vs a fresh topology without one (one split, direct store), overwrite and accumulate
@pytest.mark.parametrize("accumulate", [False, True])
@pytest.mark.parametrize("workspace", [True, False])
def test_fp32_dw_split_and_direct(workspace, accumulate):
    rng = np.random.RandomState(31)
    tp = None if workspace else TP._E().Topology(0)
    fp32_dw("fp32 dW workspace=%d accumulate=%d" % (workspace, accumulate), 4, 1200, 48, 24,
            [TP._operator(rng, 1200, 1200)], single=True, split=workspace, tp=tp, accumulate=accumulate)


# nops > 0 with F > 4: term by term, term j at dw + j * dw_term_stride; accumulate, with and without a workspace
@pytest.mark.parametrize("workspace", [True, False])
def test_fp32_dw_terms(workspace):
    rng = np.random.RandomState(41)
    tp = None if workspace else TP._E().Topology(0)
    ms = [None, TP._operator(rng, 500, 500), TP._operator(rng, 500, 500, width=11)]
    fp32_dw("fp32 dW nops=3 workspace=%d" % workspace, 3, 500, 24, 48, ms, split=workspace, tp=tp, accumulate=True)
