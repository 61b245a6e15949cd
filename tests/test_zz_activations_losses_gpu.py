"""The reference's `--activation b1relu|b1tanh` and `--loss l2|huber` on the GPU.

- kernel cases against float64 NumPy / SciPy, within 1e-4 of max |truth|: the tanh forward (CAPE_ACT_TANH) and its
  backward given the output (CAPE_EPI_TANHGRAD) in every kernel family that has epilogues -- conv_wg_kernel (fused,
  plain-operand, BN 128, two accumulators at BN 64, the pass-through instantiation), ellconv_kernel (tensor cores off:
  partial column tiles, scalar columns, F not a multiple of 4), thin_fwd_kernel, thinout_combine_kernel and cape_apply
  -- each checked for the kernel instance that ran (the tanh instantiations where there are such); and the paths
  without tanh refusing it before any launch;
- cape_recon_losses_ex against float64 for L1, L2 and Huber with residuals at 0, at +-delta and on both sides of it;
  kind L1 bit-identical to cape_recon_losses;
- the full update of CapeNetwork against the oracle (tests/options_oracle.py) for every case of
  tests/golden/ref_models_golden_5.npz / _6.npz, eager and from the captured graphs, and against those files directly;
  one update at batch 64 of the affine b1tanh + Huber model.

The file name sorts after every other GPU test file (see tests/test_resblock_encoder_gpu.py for why that matters)."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))

import make_ref_golden_options as G5  # noqa: E402
import options_oracle as OO  # noqa: E402
import parity  # noqa: E402
import resblock_oracle as R  # noqa: E402
import test_gpu_thin_paths as TP  # noqa: E402
import test_resblock_encoder_gpu as RG  # noqa: E402

pytestmark = pytest.mark.gpu

TAGS = ["affine_tanh_huber", "affine_relu_l2", "default_tanh_l2"]


# =====================================================================================================================
# conv epilogues through cape_cheb_fwd / cape_apply
# =====================================================================================================================
def conv_case(N, rows_out, ncols, specs, *, epi, passes=(), plain_only=False, shared_src=False, seed=0):
    """specs: (F, m, w2) per contracted term, m a scipy operator [rows_out x src_rows] or None (identity), w2: the term
    also feeds a second accumulator (which a LINEAR / TANHGRAD epilogue does not read).  passes: operators of
    pass-through terms (F = ncols, added to accumulator 0).  epi: "tanh" (LINEAR + bias + tanh) or "tanhgrad" (aux =
    the output of a tanh).  shared_src: every term reads the first term's source.  Returns (kernel names, relative
    error against float64)."""
    E, dev, tp = TP._E(), TP._dev(), TP._tp()
    rng = np.random.RandomState(seed)
    acc = np.zeros((N, rows_out, ncols))
    terms = []
    src_d = None
    for F, m, w2 in specs:
        src_rows = rows_out if m is None else m.shape[1]
        if not (shared_src and src_d is not None):
            src = rng.normal(size=(N, src_rows, F)).astype(np.float32)
            src_d = torch.from_numpy(src).to(dev)
        w = rng.normal(0, 1 / np.sqrt(F), size=(F, ncols)).astype(np.float32)
        acc += TP._apply(m, src) @ w.astype(np.float64)
        t = dict(src=src_d, op=TP._op_id(tp, m), F=F, src_rows=src_rows, src_stride=F,
                 w=None if plain_only else torch.from_numpy(w).to(dev), w_stride=0 if plain_only else ncols,
                 wT=torch.from_numpy(np.ascontiguousarray(w.T)).to(dev), wT_stride=F)
        if w2:
            v = rng.normal(0, 1 / np.sqrt(F), size=(F, ncols)).astype(np.float32)
            t.update(w2=torch.from_numpy(v).to(dev), w2_stride=ncols,
                     w2T=torch.from_numpy(np.ascontiguousarray(v.T)).to(dev), w2T_stride=F)
        terms.append(t)
    for m in passes:
        src_rows = rows_out if m is None else m.shape[1]
        src = rng.normal(size=(N, src_rows, ncols)).astype(np.float32)
        acc += TP._apply(m, src)
        terms.append(dict(src=torch.from_numpy(src).to(dev), op=TP._op_id(tp, m), F=ncols, src_rows=src_rows,
                          src_stride=ncols, w=None, w_stride=0))
    kw = {}
    if epi == "tanh":
        b = rng.normal(size=ncols).astype(np.float32)
        want = np.tanh(acc + b)
        kw = dict(epilogue=E.EPI_LINEAR, act=E.ACT_TANH, bias=torch.from_numpy(b).to(dev))
    else:
        aux = np.tanh(rng.normal(size=(N, rows_out, ncols))).astype(np.float32)
        want = acc * (1.0 - aux.astype(np.float64) ** 2)
        kw = dict(epilogue=E.EPI_TANHGRAD, aux=torch.from_numpy(aux).to(dev))
    out = torch.full((N, rows_out, ncols), float("nan"), device=dev)
    names = TP._traced(lambda: E.cheb_call(tp, N, rows_out, ncols, terms, out, plain_only=plain_only, **kw),
                       lambda: out.fill_(float("nan")))
    got = out.cpu().numpy()
    assert np.isfinite(got).all()
    return names, TP._rel(got.astype(np.float64), want)


def _run(case, kernel, *args, tc=True, **kw):
    with TP._knobs(tc=tc):
        names, err = conv_case(*args, **kw)
    assert TP._ran(names, kernel), (case, names, kernel)
    TP._report(case, err)
    assert err < parity.TOL, (case, err)


EPIS = ["tanh", "tanhgrad"]


@pytest.mark.parametrize("epi", EPIS)
@pytest.mark.parametrize("ncols", [128, 64, 96])
def test_conv_wg_fused(epi, ncols):
    """Two gathered terms of 64 channels: conv_wg_kernel at BN 128 (ncols 128; 96: a partial column tile) and 64."""
    rng = np.random.RandomState(ncols)
    specs = [(64, TP._operator(rng, 300, 300), False), (64, TP._operator(rng, 300, 300), False)]
    bn = 128 if ncols > 64 else 64
    _run("conv_wg fused %s ncols=%d" % (epi, ncols), "conv_wg_kernel<%d, false, false, true>" % bn, 2, 300, ncols,
         specs, epi=epi, seed=ncols)


@pytest.mark.parametrize("epi", EPIS)
def test_conv_wg_dual(epi):
    """A term with a second accumulator: conv_wg_kernel<64, true> (BN 64, one chunk accumulator)."""
    rng = np.random.RandomState(5)
    specs = [(64, TP._operator(rng, 257, 257), True), (32, None, False)]
    _run("conv_wg dual %s" % epi, "conv_wg_kernel<64, true, false, true>", 2, 257, 128, specs, epi=epi, seed=5)


@pytest.mark.parametrize("epi", EPIS)
@pytest.mark.parametrize("ncols", [64, 128])
def test_conv_wg_pass(epi, ncols):
    """Pass-through terms (the residual encoder's conv2 + skip): the PASS instantiation."""
    rng = np.random.RandomState(ncols + 1)
    specs = [(64, TP._operator(rng, 200, 200), False), (64, None, False)]
    passes = [TP._operator(rng, 200, 400), None]
    _run("conv_wg pass %s ncols=%d" % (epi, ncols), "conv_wg_kernel<%d, false, true, true>" % ncols, 2, 200, ncols,
         specs, epi=epi, passes=passes, seed=ncols)


@pytest.mark.parametrize("epi", EPIS)
@pytest.mark.parametrize("plain_only", [False, True])
def test_conv_wg_plain_operands(epi, plain_only):
    """All operators identity: the plain-operand (TMA) launch of conv_wg_kernel, with and without plain_only."""
    specs = [(48, None, False), (32, None, False)]
    _run("conv_wg plain %s plain_only=%d" % (epi, plain_only), "conv_wg_kernel<128, false, false, true>", 3, 250, 112,
         specs, epi=epi, plain_only=plain_only, seed=7)


@pytest.mark.parametrize("epi", EPIS)
@pytest.mark.parametrize("ncols,F", [(20, 13), (30, 13), (100, 24), (48, 6)])
def test_ellconv_kernel(epi, ncols, F):
    """Tensor cores off: ellconv_kernel with partial column tiles (30, 100), scalar columns (30) and F not a multiple
    of 4 (13, 6)."""
    rng = np.random.RandomState(ncols + F)
    specs = [(F, TP._operator(rng, 203, 203), False), (F, None, False)]
    _run("ellconv %s ncols=%d F=%d" % (epi, ncols, F), "ellconv_kernel<%d, false, false>" % (32 if ncols <= 32 else 64),
         3, 203, ncols, specs, epi=epi, tc=False, seed=F)


@pytest.mark.parametrize("epi", EPIS)
def test_ellconv_kernel_pass(epi):
    rng = np.random.RandomState(9)
    specs = [(24, TP._operator(rng, 150, 150), False)]
    _run("ellconv pass %s" % epi, "ellconv_kernel<64, false, true>", 2, 150, 40, specs, epi=epi,
         passes=[TP._operator(rng, 150, 300)], tc=False, seed=9)


@pytest.mark.parametrize("epi", EPIS)
@pytest.mark.parametrize("ncols", [64, 18])
def test_thin_fwd(epi, ncols):
    """3-channel inputs: thin_fwd_kernel, float4 (64) and scalar (18) columns."""
    rng = np.random.RandomState(ncols)
    specs = [(3, TP._operator(rng, 400, 400), False), (3, None, False)]
    _run("thin_fwd %s ncols=%d" % (epi, ncols), "thin_fwd_kernel<true>", 2, 400, ncols, specs, epi=epi, seed=ncols)


@pytest.mark.parametrize("ncols", [3, 1])
def test_thinout_tanh(ncols):
    """<= 4 output columns: thinout_project_kernel + thinout_combine_kernel (LINEAR only)."""
    rng = np.random.RandomState(ncols)
    m = TP._operator(rng, 300, 300)
    specs = [(64, None, False), (64, m, False)]
    _run("thinout tanh ncols=%d" % ncols, "thinout_combine_kernel", 2, 300, ncols, specs, epi="tanh", shared_src=True,
         seed=ncols)


@pytest.mark.parametrize("epi", EPIS)
@pytest.mark.parametrize("ncols", [64, 12])
def test_apply(epi, ncols):
    E, dev, tp = TP._E(), TP._dev(), TP._tp()
    rng = np.random.RandomState(ncols)
    N, rows, src_rows = 3, 333, 500
    ms = [TP._operator(rng, rows, src_rows), TP._operator(rng, rows, src_rows)]
    acc = np.zeros((N, rows, ncols))
    terms = []
    for m in ms:
        src = rng.normal(size=(N, src_rows, ncols)).astype(np.float32)
        acc += TP._apply(m, src)
        terms.append(dict(src=torch.from_numpy(src).to(dev), op=TP._op_id(tp, m), src_rows=src_rows, src_stride=ncols))
    if epi == "tanh":
        b = rng.normal(size=ncols).astype(np.float32)
        want = np.tanh(acc + b)
        kw = dict(act=E.ACT_TANH, bias=torch.from_numpy(b).to(dev))
    else:
        aux = np.tanh(rng.normal(size=(N, rows, ncols))).astype(np.float32)
        want = acc * (1.0 - aux.astype(np.float64) ** 2)
        kw = dict(epilogue=E.EPI_TANHGRAD, aux=torch.from_numpy(aux).to(dev))
    out = torch.full((N, rows, ncols), float("nan"), device=dev)
    names = TP._traced(lambda: E.apply_call(tp, N, rows, ncols, terms, out, **kw), lambda: out.fill_(float("nan")))
    assert TP._ran(names, "apply_kernel<false, true>"), names
    err = TP._rel(out.cpu().numpy().astype(np.float64), want)
    TP._report("apply %s ncols=%d" % (epi, ncols), err)
    assert err < parity.TOL


def _refused(fn, out, match):
    from cape_b200 import _lib
    lib = TP._lib()
    torch.cuda.synchronize()
    n0 = lib.cape_launch_count()
    with pytest.raises(_lib.CapeError, match=match):
        fn()
    torch.cuda.synchronize()
    assert lib.cape_launch_count() == n0
    assert bool((out == 7.0).all())


@pytest.mark.parametrize("epi", EPIS)
def test_fp32_two_accumulators_refuse_tanh(epi):
    """ellconv_kernel with two accumulators has no tanh epilogues: with tensor cores off such a call fails before any
    launch and leaves its output alone."""
    E, dev, tp = TP._E(), TP._dev(), TP._tp()
    N, rows, F, ncols = 2, 100, 32, 64
    w = torch.randn(F, ncols, device=dev)
    t = dict(src=torch.randn(N, rows, F, device=dev), op=-1, F=F, src_rows=rows, src_stride=F, w=w, w_stride=ncols,
             w2=w, w2_stride=ncols)
    out = torch.full((N, rows, ncols), 7.0, device=dev)
    kw = (dict(act=E.ACT_TANH) if epi == "tanh" else
          dict(epilogue=E.EPI_TANHGRAD, aux=torch.zeros(N, rows, ncols, device=dev)))
    with TP._knobs(tc=False):
        _refused(lambda: E.cheb_call(tp, N, rows, ncols, [t], out, **kw), out, "tanh")


def test_unknown_activation_and_dense_tanh_are_refused():
    """An activation id past CAPE_ACT_TANH, and tanh on the dense layers (cape_gemm implements none / leaky / relu)."""
    E, dev, tp = TP._E(), TP._dev(), TP._tp()
    N, rows, F, ncols = 2, 100, 32, 64
    t = dict(src=torch.randn(N, rows, F, device=dev), op=-1, F=F, src_rows=rows, src_stride=F,
             w=torch.randn(F, ncols, device=dev), w_stride=ncols)
    out = torch.full((N, rows, ncols), 7.0, device=dev)
    _refused(lambda: E.cheb_call(tp, N, rows, ncols, [t], out, act=E.ACT_TANH + 1), out, "unknown activation")
    a = [dict(src=t["src"], op=-1, src_rows=rows, src_stride=F)]
    out2 = torch.full((N, rows, F), 7.0, device=dev)
    _refused(lambda: E.apply_call(tp, N, rows, F, a, out2, act=E.ACT_TANH + 1), out2, "unknown activation")
    c = torch.full((8, 16), 7.0, device=dev)
    _refused(lambda: E.gemm(tp, torch.randn(8, 4, device=dev), torch.randn(4, 16, device=dev), c, act=E.ACT_TANH), c,
             "cape_gemm implements")


# =====================================================================================================================
# cape_recon_losses_ex
# =====================================================================================================================
DELTA = np.float32(0.1)


def _loss_case(N, rows, seed):
    """pred / gt with residuals exactly 0, +-delta, just inside and outside it, small and large; a random graph."""
    import scipy.sparse as sp
    rng = np.random.RandomState(seed)
    special = np.array([0, DELTA, -DELTA, np.nextafter(DELTA, 0), -np.nextafter(DELTA, 0), np.nextafter(DELTA, 1),
                        -np.nextafter(DELTA, 1), 0.05, -0.05, 2.0, -2.0], np.float32)
    d = rng.normal(0, 0.2, size=(N, rows, 3)).astype(np.float32)
    d.reshape(-1)[:special.size] = special
    gt = rng.normal(size=(N, rows, 3)).astype(np.float32)
    gt.reshape(-1)[:special.size] = 0.0
    pred = (gt + d).astype(np.float32)
    pred.reshape(-1)[:special.size] = special
    a = sp.random(rows, rows, density=6.0 / rows, random_state=seed, format="csr")
    a = ((a + a.T) > 0).astype(np.float32)
    a.setdiag(0)
    a.eliminate_zeros()
    return pred, gt, sp.csr_matrix(a)


def _loss_truth(kind, pred, gt, adj, lam_r, lam_e):
    p, g = pred.astype(np.float64), gt.astype(np.float64)
    d = p - g
    cnt = d.size
    delta = float(DELTA)
    if kind == "l1":
        val, gr = np.abs(d), np.sign(d)
    elif kind == "l2":
        val, gr = d * d, 2 * d
    else:
        q = np.minimum(np.abs(d), delta)
        val, gr = 0.5 * q * q + delta * (np.abs(d) - q), np.clip(d, -delta, delta)
    coo = adj.tocoo()
    e = d[:, coo.row] - d[:, coo.col]
    ln = np.linalg.norm(e, axis=-1)
    n_edges = coo.nnz // 2
    edge = 0.5 * ln.sum() / (d.shape[0] * n_edges)
    ge = np.zeros_like(d)
    for n in range(d.shape[0]):
        np.add.at(ge[n], coo.row, e[n] / np.where(ln[n] > 0, ln[n], 1.0)[:, None])
    grad = lam_r * gr / cnt + lam_e * ge / (d.shape[0] * n_edges)
    return val.mean(), edge, grad


def _losses(fn_name, kind, pred, gt, adj, lam_r, lam_e, kl=None):
    E, dev, tp, lib = TP._E(), TP._dev(), TP._tp(), TP._lib()
    from cape_b200 import _lib
    N, rows = pred.shape[:2]
    op = tp.add_operator(adj)
    P, Gt = torch.from_numpy(pred).to(dev), torch.from_numpy(gt).to(dev)
    dpred = torch.zeros_like(P)
    L = torch.zeros(3, device=dev)
    mean, logvar = kl if kl is not None else (None, None)
    nz = mean.shape[1] if kl is not None else 0
    common = (E._ptr(mean), E._ptr(logvar), nz, E._ptr(dpred), E._ptr(L), E._stream())
    n_edges = adj.nnz // 2
    if fn_name == "cape_recon_losses":
        rc = lib.cape_recon_losses(tp.h, op, E._ptr(P), E._ptr(Gt), N, rows, lam_r, lam_e, n_edges, *common)
    else:
        kid = {"l1": E.RECON_L1, "l2": E.RECON_L2, "huber": E.RECON_HUBER}[kind]
        rc = lib.cape_recon_losses_ex(tp.h, op, E._ptr(P), E._ptr(Gt), N, rows, kid, float(DELTA), lam_r, lam_e,
                                      n_edges, *common)
    _lib.check(rc)
    torch.cuda.synchronize()
    return L.cpu().numpy(), dpred.cpu().numpy()


@pytest.mark.parametrize("kind", ["l1", "l2", "huber"])
@pytest.mark.parametrize("lam_e", [0.0, 1.0])
def test_recon_losses_vs_float64(kind, lam_e):
    pred, gt, adj = _loss_case(3, 700, 1)
    L, dpred = _losses("ex", kind, pred, gt, adj, 1.0, lam_e)
    val, edge, grad = _loss_truth(kind, pred, gt, adj, 1.0, lam_e)
    print("recon %s: value %.3e edge %.3e grad %.3e" % (kind, abs(L[0] - val) / val, abs(L[1] - edge) / edge,
                                                         TP._rel(dpred.astype(np.float64), grad)))
    assert abs(L[0] - val) <= 1e-5 * val and abs(L[1] - edge) <= 1e-5 * edge
    assert TP._rel(dpred.astype(np.float64), grad) < parity.TOL
    if kind == "huber" and lam_e == 0.0:
        # the special residuals: gradient clamp(d, +-delta) / cnt exactly where |d| reaches delta
        flat, want = dpred.reshape(-1)[:11] * pred.size, np.clip(pred.reshape(-1)[:11], -DELTA, DELTA)
        assert np.allclose(flat, want, rtol=1e-6, atol=0), (flat, want)


def test_recon_losses_l1_is_bit_identical():
    """kind L1 of cape_recon_losses_ex is cape_recon_losses: the same losses (one block: a fixed summation order) and
    the same gradient, with the KL term."""
    dev = TP._dev()
    pred, gt, adj = _loss_case(2, 100, 3)
    rng = np.random.RandomState(4)
    kl = (torch.from_numpy(rng.normal(size=(2, 18)).astype(np.float32)).to(dev),
          torch.from_numpy(rng.normal(size=(2, 18)).astype(np.float32)).to(dev))
    a = _losses("cape_recon_losses", "l1", pred, gt, adj, 0.7, 0.3, kl)
    b = _losses("ex", "l1", pred, gt, adj, 0.7, 0.3, kl)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    pred, gt, adj = _loss_case(4, 3000, 5)
    a = _losses("cape_recon_losses", "l1", pred, gt, adj, 0.7, 0.3)
    b = _losses("ex", "l1", pred, gt, adj, 0.7, 0.3)
    assert np.array_equal(a[1], b[1])


def test_recon_losses_rejects_unknown_kinds():
    from cape_b200 import _lib
    E, dev, tp, lib = TP._E(), TP._dev(), TP._tp(), TP._lib()
    pred, gt, adj = _loss_case(1, 50, 6)
    op = tp.add_operator(adj)
    P, Gt = torch.from_numpy(pred).to(dev), torch.from_numpy(gt).to(dev)
    dpred = torch.zeros_like(P)
    L = torch.zeros(3, device=dev)
    for kind, delta in ((3, 0.1), (E.RECON_HUBER, 0.0)):
        rc = lib.cape_recon_losses_ex(tp.h, op, E._ptr(P), E._ptr(Gt), 1, 50, kind, delta, 1.0, 1.0, adj.nnz // 2,
                                      None, None, 0, E._ptr(dpred), E._ptr(L), E._stream())
        assert rc < 0
    with pytest.raises(_lib.CapeError):
        _lib.check(-1)


# =====================================================================================================================
# the network
# =====================================================================================================================
def _cfg(tag):
    return next(c for t, c, n, s in G5.configs() if t == tag)


@pytest.mark.parametrize("mode", ["eager", "graph"])
@pytest.mark.parametrize("tag", TAGS)
def test_update_matches_oracle(hierarchy, monkeypatch, tag, mode):
    """One update at batch 2 against the oracle's autograd: x_hat and the losses with and without the CUDA branch
    decisions imposed, every gradient, clipped update and parameter with them."""
    monkeypatch.setattr(R, "ResOracle", OO.OptOracle)
    res = R.train_step(hierarchy, _cfg(tag), N=2, use_graph=mode == "graph")
    print("%s %s: worst %s" % (tag, mode, max(res.items(), key=lambda kv: kv[1])))
    RG._assert_parity(res, tag + " " + mode)


@pytest.mark.parametrize("tag", TAGS)
def test_update_matches_the_reference_golden(hierarchy, tag):
    """x_hat, the five losses and the discriminator's post-update parameters of ref_models_golden_5.npz / _6.npz."""
    out = RG.golden_update_errors(hierarchy, G5.configs, G5.load, tag)
    assert max(out.values()) < parity.TOL, {k: v for k, v in out.items() if not v < parity.TOL}


def test_batch64_affine_tanh_huber(hierarchy, monkeypatch):
    """The benchmark's batch: its layer forms and split-K shapes, with tanh epilogues and the Huber loss."""
    monkeypatch.setattr(R, "ResOracle", OO.OptOracle)
    res = R.train_step(hierarchy, _cfg("affine_tanh_huber"), N=64)
    print("affine_tanh_huber N=64: worst %s" % (max(res.items(), key=lambda kv: kv[1]),))
    RG._assert_parity(res, "affine_tanh_huber N=64")


def test_cape_predicts_encodes_decodes_and_checkpoints(hierarchy, tmp_path):
    """Through the public CAPE class built from a config with `activation: b1tanh` and `loss: huber`: encode and
    decode against the oracle, predict reporting the Huber loss of its own predictions, a checkpoint round trip."""
    import tempfile
    from cape_b200.config_parser import model_params, parse_config
    from cape_b200.models import CAPE
    from cape_b200.synthetic import make_batch
    h = hierarchy
    fn = os.path.join(tempfile.mkdtemp(), "c.yaml")
    open(fn, "w").write("nz: 64\nnz_cond: 32\nnz_cond2: 32\naffine: 1\nlr_warmup: 1\nname: opt_test\nbatch_size: 2\n"
                        "mode: demo\nactivation: b1tanh\nloss: huber\n")
    args, _ = parse_config(["--config", fn])
    p = model_params(args)
    p["p"] = h["p"]
    m = CAPE(L=h["L"], D=h["D"], U=h["U"], L_d=h["L_d"], D_d=h["D_d"], **p)
    assert m.cfg["activation"] == "b1tanh" and m.cfg["loss"] == "huber"
    m.build_graph(m.input_num_verts, m.nn_input_channel, phase="demo")
    m.checkpoint_dir = str(tmp_path)
    params = parity.calibrated_params(m.net.specs, 11)
    m.load_weights(params)
    b = make_batch(4, 64, seed=5)
    o = OO.OptOracle(h["L"], h["D"], h["U"], h["L_d"], h["D_d"], m.cfg)
    P = {k: torch.from_numpy(v) for k, v in params.items()}
    t = torch.from_numpy
    y, y2 = o.cond_embeddings(t(b["cond_g"]), t(b["cond2_g"]), P)
    zm, zl = o.encoder(t(b["x_g"]), P)
    gm, gl, gc, gc2 = m.encode(b["x_g"], b["cond_g"], b["cond2_g"])
    assert parity.rel(gm, zm.numpy()) < 1e-4 and parity.rel(gl, zl.numpy()) < 1e-4
    z_total = np.concatenate([np.random.RandomState(0).normal(size=(4, 64)).astype(np.float32), gc, gc2], 1)
    want = o.decoder_cond_vert(t(z_total), y, y2, P).numpy()
    assert parity.vertex_l2(m.decode(z_total, gc, gc2), want) < 1e-4
    preds, recon, latent, edge = m.predict(b["x_g"], b["cond_g"], b["cond2_g"], labels=b["x_g"])
    # lib/models.py:1039,1083-1086: the last of the two batches enters the mean with weight 0
    d = preds[:2].astype(np.float64) - b["x_g"][:2]
    q = np.minimum(np.abs(d), 0.1)
    want_recon = (0.5 * q * q + 0.1 * (np.abs(d) - q)).mean() * 2 / 4
    assert abs(recon - want_recon) <= 1e-4 * want_recon, (recon, want_recon)
    before = m.net.get_params()
    m.save(7)
    m.net.set_params({k: v * 0 for k, v in before.items()})
    m.restore()
    after = m.net.get_params()
    assert all(np.array_equal(before[k], after[k]) for k in before)
