"""The reference's plain decoder (`--use_res_block_dec 0`) and `--reduce_dim 0` on the GPU: cape_gemm_ex's data-gradient
epilogues through the C ABI against float64, the kernels the plain decoder's layers launch, and CapeNetwork against the
oracle (tests/plaindec_oracle.py) and against the reference's own numbers (tests/golden/ref_models_golden_7.npz, _8).

The file name sorts after every existing GPU test file, so that in one `pytest -m gpu` process the existing tests run
after exactly the tests they ran after before, in the same process state."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))

import make_ref_golden as G  # noqa: E402
import make_ref_golden_plaindec as G7  # noqa: E402
import parity  # noqa: E402
import plaindec_oracle as PD  # noqa: E402
import test_gpu_thin_paths as TP  # noqa: E402
import test_resblock_encoder_gpu as TR  # noqa: E402

pytestmark = pytest.mark.gpu

TAGS = [t for t, _, _, _ in G7.configs()]


def _cfg(tag):
    return next(c for t, c, n, s in G7.configs() if t == tag)


# ---- cape_gemm_ex through the C ABI ---------------------------------------------------------------------------------
_GEMM_TP = []


def _gemm_tp():
    """One handle with a split-K workspace for every case of this file."""
    if not _GEMM_TP:
        E = TP._E()
        tp = E.Topology(0)
        tp.reserve_workspace(64 << 20)
        _GEMM_TP.append(tp)
    return _GEMM_TP[0]


# (M, N, K, transposed B): the FC data gradient at reduce_dim 0 (g [N, nz] @ W^T, direct store: scalar kernel for
# nz 18, vectorised for nz 64), and few-tile products with a long reduction (split-K, both kernels)
GEMM_SHAPES = {"direct-scalar": (64, 20000, 18, True), "direct-vec": (64, 20000, 64, True),
               "splitk-scalar": (18, 50, 30000, False), "splitk-vec": (64, 64, 30000, False)}


@pytest.mark.parametrize("beta", [0.0, 1.0])
@pytest.mark.parametrize("epi", ["slope0.2", "slope0", "tanhgrad"])
@pytest.mark.parametrize("shape", list(GEMM_SHAPES))
def test_gemm_ex_epilogues(shape, epi, beta):
    """C = epi(A @ B + beta C; aux) for aux with C's layout; C's rows are padded with NaN columns that must stay
    untouched, and with beta = 0 the NaN in C itself must not be read."""
    E = TP._E()
    tp = _gemm_tp()
    M, N, K, bt = GEMM_SHAPES[shape]
    rng = np.random.RandomState(M + N + K + len(epi) + int(beta))
    A = rng.randn(M, K).astype(np.float32)
    B = (rng.randn(N, K) if bt else rng.randn(K, N)).astype(np.float32) * 0.1
    aux = rng.randn(M, N).astype(np.float32)
    aux[rng.rand(M, N) < 0.01] = 0.0                          # exact zeros: the SLOPE mask takes alpha there
    if epi == "tanhgrad":
        aux = np.tanh(aux)
    c0 = rng.randn(M, N).astype(np.float32)
    pad = 4
    init = np.full((M, N + pad), np.nan, np.float32)
    if beta:
        init[:, :N] = c0
    dev = TP._dev()
    Ad, Bd, auxd = (torch.from_numpy(v).to(dev) for v in (A, B, aux))
    Cbuf = torch.from_numpy(init).to(dev)
    Bv = Bd.t() if bt else Bd
    kw = dict(epilogue=E.EPI_TANHGRAD) if epi == "tanhgrad" else dict(epilogue=E.EPI_SLOPE,
                                                                       epi_alpha=float(epi[len("slope"):]))
    E.gemm(tp, Ad, Bv, Cbuf[:, :N], beta=beta, aux=auxd, **kw)
    torch.cuda.synchronize()
    acc = A.astype(np.float64) @ (B.T if bt else B).astype(np.float64) + beta * c0.astype(np.float64)
    a64 = aux.astype(np.float64)
    want = acc * (1 - a64 * a64) if epi == "tanhgrad" else acc * np.where(a64 > 0, 1.0, kw["epi_alpha"])
    got = Cbuf.cpu().numpy()
    assert np.isnan(got[:, N:]).all(), "wrote into the padding columns"
    assert np.isfinite(got[:, :N]).all()
    err = TP._rel(got[:, :N].astype(np.float64), want)
    TP._report("gemm_ex %s %s beta=%g" % (shape, epi, beta), err)
    assert err < 1e-4, err


def test_gemm_ex_linear_is_cape_gemm():
    """Epilogue LINEAR: the same call as cape_gemm, bit for bit."""
    E = TP._E()
    tp = _gemm_tp()
    lib = TP._lib()
    dev = TP._dev()
    A, B = torch.randn(64, 300, device=dev), torch.randn(300, 70, device=dev)
    c1, c2 = torch.zeros(64, 70, device=dev), torch.zeros(64, 70, device=dev)
    E.gemm(tp, A, B, c1)
    E.check(lib.cape_gemm_ex(tp.h, 64, 70, 300, E._ptr(A), 300, 1, E._ptr(B), 70, 1, E._ptr(c2), 70, None,
                             E.ACT_NONE, 0.2, 1.0, 0.0, E.EPI_LINEAR, 0.0, None, 0, E._stream()))
    torch.cuda.synchronize()
    assert torch.equal(c1, c2)


def test_gemm_ex_refusals():
    from cape_b200 import _lib
    E = TP._E()
    tp = _gemm_tp()
    dev = TP._dev()
    A, B, C = torch.randn(4, 8, device=dev), torch.randn(8, 4, device=dev), torch.zeros(4, 4, device=dev)
    for epi, aux in ((E.EPI_SLOPE, None), (E.EPI_AFFINE, C), (E.EPI_DUALMASK, C), (17, C)):
        with pytest.raises(_lib.CapeError):
            E.check(tp.lib.cape_gemm_ex(tp.h, 4, 4, 8, E._ptr(A), 8, 1, E._ptr(B), 4, 1, E._ptr(C), 4, None,
                                        E.ACT_NONE, 0.2, 1.0, 0.0, epi, 0.2, E._ptr(aux), 4, E._stream()))


# ---- the plain decoder's launches -----------------------------------------------------------------------------------
@pytest.mark.parametrize("tag", ["plain_nz18", "plain_nz64_rd0_tanh_l2"])
def test_plain_decoder_kernel_census(hierarchy, tag):
    """Every dec/conv* forward and data-gradient launch takes the tensor-core kernels: none falls back to the fp32
    ellconv_kernel.  Prints the kernels each launch ran and the forms choose_forms picked."""
    from cape_b200.network import CapeNetwork
    from cape_b200.synthetic import make_batch
    h = hierarchy
    cfg = _cfg(tag)
    N = 2
    net = CapeNetwork(h["L"], h["D"], h["U"], h["L_d"], h["D_d"], cfg, N)
    tb = {k: torch.from_numpy(v) for k, v in make_batch(N, cfg["nz"], seed=1).items()}
    net.set_inputs(tb["x_g"], tb["cond_g"], tb["cond2_g"], tb["eps"], tb["x_d"], tb["cond_d"], tb["cond2_d"])
    _, epi, alpha = net.brelu
    with TP._knobs(tc=True):
        net.train_step(update=False)
        torch.cuda.synchronize()
        for i, l in enumerate(net.dec):
            x = net.dec_act[i - 1] if i else net.dec_h0
            fwd = TP._traced(lambda: l.fwd(x, net.ycat_g, net.dec_act[i]), lambda: None)
            kw = dict(dx_epi=epi, dx_aux=x, dx_alpha=alpha) if i else {}
            dx = net.g_dec[i - 1] if i else net.g_dec_h0
            bwd = TP._traced(lambda: (l.bwd(x, net.ycat_g, net.g_dec[i], dx=dx, dycat=net.d_ycat, **kw), net.join_dw()),
                             lambda: None)
            print("%s (%s, fwd %s, dx %s, dW %s): fwd %s | bwd %s" % (l.name, "%d->%d x%d rows %d->%d" % (
                l.F, l.Fout, l.K, l.site.rows_in, l.site.rows_out), l.fwd_mode, l.dx_mode, l.dw_mode, fwd, bwd))
            assert not TP._ran(fwd, "ellconv_kernel") and not TP._ran(bwd, "ellconv_kernel"), (l.name, fwd, bwd)
            assert TP._ran(fwd, "conv_wg_kernel") and TP._ran(bwd, "conv_wg_kernel"), (l.name, fwd, bwd)
        net.small.flush()
        torch.cuda.synchronize()


# ---- the network ------------------------------------------------------------------------------------------------------
def _fc_scale(cfg, N):
    """The FC kernels' scale for the comparison: at reduce_dim 0 the FC layers read 8x more features, and at batch 64
    the larger encoder outputs need the smaller scale test_resblock_encoder_gpu.py uses (the KL term's exp() turns fp32
    rounding of log-variances of a few units into 1e-4 of the loss in any fp32 implementation)."""
    return 0.01 if (cfg["reduce_dim"] <= 0 or N > 2) else 0.05


@pytest.mark.parametrize("mode", ["eager", "graph"])
@pytest.mark.parametrize("tag", TAGS)
def test_update_matches_oracle(hierarchy, tag, mode):
    cfg = _cfg(tag)
    res = PD.train_step(hierarchy, cfg, N=2, use_graph=mode == "graph", fc_scale=_fc_scale(cfg, 2))
    print("%s %s: worst %s" % (tag, mode, max(res.items(), key=lambda kv: kv[1])))
    TR._assert_parity(res, "%s %s" % (tag, mode))


@pytest.mark.parametrize("tag", TAGS)
def test_update_at_batch_64_matches_oracle(hierarchy, tag):
    cfg = _cfg(tag)
    res = PD.train_step(hierarchy, cfg, N=64, use_graph=True, fc_scale=_fc_scale(cfg, 64))
    print("%s N=64: worst %s" % (tag, max(res.items(), key=lambda kv: kv[1])))
    TR._assert_parity(res, "%s N=64" % tag)


@pytest.mark.parametrize("tag", TAGS)
def test_update_matches_the_reference_golden(hierarchy, tag):
    """The update ref_models_golden_7.npz / _8.npz hold, on the CUDA path."""
    out = TR.golden_update_errors(hierarchy, G7.configs, G7.load, tag)
    assert max(out.values()) < parity.TOL, {k: v for k, v in out.items() if not v < parity.TOL}


@pytest.mark.parametrize("tag", ["plain_nz64_rd0_tanh_l2", "default_rd0"])
def test_patch_order_at_reduce_dim_0(hierarchy, tag):
    """reorder=True without the 1x1 convs: the permutation is folded into the last encoder layer's output tables and
    the first decoder layer's input tables, so the FC rows keep the reference's numbering."""
    cfg = _cfg(tag)
    res = PD.train_step(hierarchy, cfg, N=2, reorder=True, fc_scale=_fc_scale(cfg, 2))
    print("%s reorder: worst %s" % (tag, max(res.items(), key=lambda kv: kv[1])))
    TR._assert_parity(res, tag + " reorder")


def test_plain_decoder_on_a_generated_4_layer_hierarchy(hierarchy):
    """`--num_conv_layers 4 --ds_factor 4`: the plain decoder's un-pooling layers on operators cape_b200.mesh_sampling
    generates from the template mesh."""
    from cape_b200 import main as M
    L, D, U, p = M.build_hierarchy(num_conv_layers=4, ds_factor=4)
    h = dict(L=L, D=D, U=U, p=p, L_d=hierarchy["L_d"], D_d=hierarchy["D_d"])
    cfg = dict(_cfg("plain_nz18"), F=[64, 128, 128, 64], K=[2] * 4)
    res = PD.train_step(h, cfg, N=2)
    print("4-layer ds 4 %s: worst %s" % (p, max(res.items(), key=lambda kv: kv[1])))
    TR._assert_parity(res, "4-layer")


@pytest.mark.parametrize("tag", ["plain_nz18", "plain_nz64_rd0_tanh_l2"])
def test_encode_decode_predict(hierarchy, tag):
    from cape_b200.models import CAPE
    from cape_b200.synthetic import make_batch
    h = hierarchy
    cfg = _cfg(tag)
    kw = dict(G.reference_kwargs(cfg, dict(h, p=h["p"]), 4), activation=cfg["activation"])
    m = CAPE(**kw)
    m.build_graph(m.input_num_verts, m.nn_input_channel, phase="demo")
    params = parity.calibrated_params(m.net.specs, 11, _fc_scale(cfg, 2))
    m.load_weights(params)
    n = 6
    b = make_batch(n, cfg["nz"], seed=5)
    o = PD.PlainDecOracle(h["L"], h["D"], h["U"], h["L_d"], h["D_d"], cfg)
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


@pytest.mark.parametrize("tag", ["plain_nz18", "plain_nz64_rd0_tanh_l2"])
def test_tensorflow_checkpoint_restores_by_name(hierarchy, tmp_path, tag):
    from cape_b200 import tf_checkpoint
    from cape_b200.network import CapeNetwork
    h = hierarchy
    net = CapeNetwork(h["L"], h["D"], h["U"], h["L_d"], h["D_d"], _cfg(tag), 1)
    params = parity.calibrated_params(net.specs, 3)
    prefix = str(tmp_path / "model.ckpt-5")
    tf_checkpoint.write_checkpoint(prefix, dict(params, global_step=np.asarray(5, np.int64)))
    names = {n for n, _, _ in tf_checkpoint.list_variables(prefix)}
    assert {n for n in names if "decoder_conv" in n} == {n for n in net.specs if "decoder_conv" in n}
    net.set_params(tf_checkpoint.read_checkpoint(prefix, names=list(net.specs)))
    got = net.get_params()
    assert all(np.array_equal(got[k], params[k]) for k in params)
