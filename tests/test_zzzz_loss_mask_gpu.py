"""The reference's `--loss_mask binary` on the GPU.

- cape_recon_losses_w against float64 for L1, L2 and Huber, with the shipped mask and with random positive weights,
  residuals at 0, at +-delta and on both sides of it, N in {1, 2, 64}; an all-ones mask bit-identical to
  cape_recon_losses_ex;
- the full update of CapeNetwork against the oracle (tests/lossmask_oracle.py) for every case of
  tests/golden/ref_models_golden_9.npz / _10.npz: at batch 2 eager, graph-replayed and in patch order (`reorder`: the
  mask is indexed in the reference's vertex numbering, which x_hat keeps), at batch 64 graph-replayed, and against those
  files directly;
- CAPE.predict / evaluate on a padded last batch reporting the masked term, a TensorFlow checkpoint round trip of a
  masked model, `python -m cape_b200.main --loss_mask binary` in train and test mode, and (with two GPUs) one
  data-parallel step against the single-GPU step on the global batch.

The file name sorts after every other GPU test file (see tests/test_resblock_encoder_gpu.py for why that matters)."""
import os
import socket
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))

import make_ref_golden as G  # noqa: E402
import make_ref_golden_lossmask as G9  # noqa: E402
import lossmask_oracle as LM  # noqa: E402
import parity  # noqa: E402
import resblock_oracle as R  # noqa: E402
import test_gpu_thin_paths as TP  # noqa: E402
import test_resblock_encoder_gpu as RG  # noqa: E402
import test_zz_activations_losses_gpu as ZZ  # noqa: E402

pytestmark = pytest.mark.gpu

TAGS = ["affine_l1_mask", "nz18_l2_mask", "default_huber_mask"]
KINDS = ["l1", "l2", "huber"]


# =====================================================================================================================
# cape_recon_losses_w
# =====================================================================================================================
def _mask(which, rows, seed=0):
    from cape_b200 import topology as T
    if which == "shipped":
        return T.loss_mask_binary()
    if which == "ones":
        return np.ones(rows, np.float32)
    return np.random.RandomState(seed).uniform(0.05, 2.0, size=rows).astype(np.float32)


def _truth(kind, pred, gt, adj, m, lam_r, lam_e):
    """float64 (recon, edge, dpred) of the weighted reconstruction term and the unweighted edge term."""
    _, edge, g_unw = ZZ._loss_truth(kind, pred, gt, adj, 0.0, lam_e)
    d = pred.astype(np.float64) - gt.astype(np.float64)
    w = m.astype(np.float64)[None, :, None]
    delta = float(ZZ.DELTA)
    if kind == "l1":
        val, gr = np.abs(d), np.sign(d)
    elif kind == "l2":
        val, gr = d * d, 2 * d
    else:
        q = np.minimum(np.abs(d), delta)
        val, gr = 0.5 * q * q + delta * (np.abs(d) - q), np.clip(d, -delta, delta)
    cnt = 3.0 * d.shape[0] * m.astype(np.float64).sum()
    return (w * val).sum() / cnt, edge, g_unw + lam_r * w * gr / cnt


def _weighted(kind, pred, gt, adj, m, lam_r, lam_e, kl=None, weighted=True):
    """(losses, dpred) of cape_recon_losses_w (weighted) or cape_recon_losses_ex, through engine.recon_losses."""
    E, dev, tp = TP._E(), TP._dev(), TP._tp()
    N, rows = pred.shape[:2]
    op = tp.add_operator(adj)
    P, Gt = torch.from_numpy(pred).to(dev), torch.from_numpy(gt).to(dev)
    dpred = torch.zeros_like(P)
    L = torch.zeros(3, device=dev)
    mean, logvar = kl if kl is not None else (None, None)
    nz = mean.shape[1] if kl is not None else 0
    kid = {"l1": E.RECON_L1, "l2": E.RECON_L2, "huber": E.RECON_HUBER}[kind]
    mk = dict(mask=torch.from_numpy(m).to(dev), mask_sum=float(m.astype(np.float64).sum())) if weighted else {}
    E.recon_losses(tp, op, P, Gt, N, rows, kid, lam_r, lam_e, adj.nnz // 2, mean, logvar, nz, dpred, L, **mk)
    torch.cuda.synchronize()
    return L.cpu().numpy(), dpred.cpu().numpy()


@pytest.mark.parametrize("N", [1, 2, 64])
@pytest.mark.parametrize("which", ["shipped", "random"])
@pytest.mark.parametrize("kind", KINDS)
def test_recon_losses_w_vs_float64(kind, which, N):
    """Loss and gradient within 1e-6 of the truth's max, on the SMPL vertex count with a random neighbour graph."""
    pred, gt, adj = ZZ._loss_case(N, 6890, N)
    m = _mask(which, 6890, seed=N)
    L, dpred = _weighted(kind, pred, gt, adj, m, 0.7, 0.3)
    val, edge, grad = _truth(kind, pred, gt, adj, m, 0.7, 0.3)
    e_val, e_edge = abs(L[0] - val) / val, abs(L[1] - edge) / edge
    e_grad = TP._rel(dpred.astype(np.float64), grad)
    print("recon_w %s %s N=%d: value %.2e edge %.2e dpred %.2e" % (kind, which, N, e_val, e_edge, e_grad))
    assert e_val <= 1e-6 and e_grad <= 1e-6
    assert e_edge <= 1e-5                     # the unweighted edge term, as cape_recon_losses_ex's tests bound it
    if N == 1:
        # the special residuals on vertices 0-3, without the edge term: the weighted gradient of each kind exactly
        # where it changes form (an L1 residual of exactly 0 gets gradient 0; Huber's is clamp(d, +-delta))
        _, dpred = _weighted(kind, pred, gt, adj, m, 0.7, 0.0)
        _, _, grad = _truth(kind, pred, gt, adj, m, 0.7, 0.0)
        got, want = dpred.reshape(-1)[:11], grad.reshape(-1)[:11]
        assert np.allclose(got, want, rtol=1e-6, atol=0), (got, want)
        if kind == "l1":
            assert got[0] == 0.0


@pytest.mark.parametrize("kind", KINDS)
def test_all_ones_mask_is_bit_identical_to_the_unweighted_call(kind):
    """Weights 1 with their sum `rows` are the unweighted term: the same losses (one block: a fixed summation order),
    KL included, and the same gradient on a many-block problem."""
    dev = TP._dev()
    rng = np.random.RandomState(4)
    kl = (torch.from_numpy(rng.normal(size=(2, 18)).astype(np.float32)).to(dev),
          torch.from_numpy(rng.normal(size=(2, 18)).astype(np.float32)).to(dev))
    pred, gt, adj = ZZ._loss_case(2, 100, 3)
    ones = _mask("ones", 100)
    a = _weighted(kind, pred, gt, adj, ones, 0.7, 0.3, kl)
    b = _weighted(kind, pred, gt, adj, ones, 0.7, 0.3, kl, weighted=False)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    pred, gt, adj = ZZ._loss_case(4, 6890, 5)
    ones = _mask("ones", 6890)
    a = _weighted(kind, pred, gt, adj, ones, 0.7, 0.3)
    b = _weighted(kind, pred, gt, adj, ones, 0.7, 0.3, weighted=False)
    assert np.array_equal(a[1], b[1])


def test_recon_losses_w_refuses_bad_weights():
    from cape_b200 import _lib
    E, dev, tp, lib = TP._E(), TP._dev(), TP._tp(), TP._lib()
    pred, gt, adj = ZZ._loss_case(1, 50, 6)
    op = tp.add_operator(adj)
    P, Gt = torch.from_numpy(pred).to(dev), torch.from_numpy(gt).to(dev)
    dpred = torch.zeros_like(P)
    L = torch.zeros(3, device=dev)
    w = torch.ones(50, device=dev)
    torch.cuda.synchronize()
    n0 = lib.cape_launch_count()
    for ptr, s in ((None, 50.0), (E._ptr(w), 0.0), (E._ptr(w), -1.0), (E._ptr(w), float("nan"))):
        rc = lib.cape_recon_losses_w(tp.h, op, E._ptr(P), E._ptr(Gt), 1, 50, E.RECON_L1, 0.1, 1.0, 1.0, adj.nnz // 2,
                                     ptr, s, None, None, 0, E._ptr(dpred), E._ptr(L), E._stream())
        assert rc < 0
    torch.cuda.synchronize()
    assert lib.cape_launch_count() == n0
    with pytest.raises(_lib.CapeError, match="vertex weights"):
        _lib.check(rc)


# =====================================================================================================================
# the network
# =====================================================================================================================
def _cfg(tag):
    return next(c for t, c, n, s in G9.configs() if t == tag)


@pytest.mark.parametrize("mode", ["eager", "graph", "reorder"])
@pytest.mark.parametrize("tag", TAGS)
def test_update_matches_oracle(hierarchy, monkeypatch, tag, mode):
    """One update at batch 2 against the oracle's autograd: x_hat and the losses with and without the CUDA branch
    decisions imposed, every gradient, clipped update and parameter with them."""
    monkeypatch.setattr(R, "ResOracle", LM.MaskOracle)
    res = R.train_step(hierarchy, _cfg(tag), N=2, use_graph=mode == "graph", reorder=mode == "reorder")
    print("%s %s: worst %s" % (tag, mode, max(res.items(), key=lambda kv: kv[1])))
    if tag == "default_huber_mask":
        # The default config has lambda_edge 0, so the Huber term alone sets the scale of dpred; below delta its
        # gradient is the residual itself and carries x_hat's absolute fp32 rounding, scaled by 1 / delta.  The
        # per-vertex bias gradient of `outputs` (dpred summed over the batch) is that ill-conditioned in any fp32
        # implementation: the oracle in fp32 and in fp64 differ on it by 2.6e-4 at this batch.
        for k in ("grad ", "clipped-update "):
            assert res.pop(k + "generator/decoder/outputs/bias") < 5e-4, k
    RG._assert_parity(res, tag + " " + mode)


@pytest.mark.parametrize("tag", TAGS)
def test_update_at_batch_64_matches_oracle(hierarchy, monkeypatch, tag):
    """The benchmark's batch through the captured graphs.  The default model's residual encoder takes the smaller fc
    scale of tests/test_resblock_encoder_gpu.py's batch-64 test, for the reason given there."""
    monkeypatch.setattr(R, "ResOracle", LM.MaskOracle)
    fc_scale = 0.01 if tag.startswith("default") else 0.05
    res = R.train_step(hierarchy, _cfg(tag), N=64, use_graph=True, fc_scale=fc_scale)
    print("%s N=64: worst %s" % (tag, max(res.items(), key=lambda kv: kv[1])))
    RG._assert_parity(res, tag + " N=64")


@pytest.mark.parametrize("tag", TAGS)
def test_update_matches_the_reference_golden(hierarchy, tag):
    """x_hat, the five losses and the discriminator's post-update parameters of ref_models_golden_9.npz / _10.npz."""
    out = RG.golden_update_errors(hierarchy, G9.configs, G9.load, tag)
    assert max(out.values()) < parity.TOL, {k: v for k, v in out.items() if not v < parity.TOL}


def _masked_model(h, N, tag="affine_l1_mask"):
    from cape_b200.models import CAPE
    cfg = _cfg(tag)
    m = CAPE(**dict(G.reference_kwargs(cfg, dict(h, p=h["p"]), N), loss_mask="binary"))
    m.build_graph(m.input_num_verts, m.nn_input_channel, phase="demo")
    return m, cfg


def test_predict_and_evaluate_report_the_masked_term(hierarchy):
    """Six meshes at batch 4: the second batch is zero-padded.  The reported term is calc_mean of the per-batch masked
    terms (lib/models.py:1083-1086, which gives the padded last batch weight 0), each the oracle's masked term of its
    batch; the padded batch's own term covers all four rows, padding included, with the denominator 3 * 4 * sum(m)."""
    from cape_b200.synthetic import make_batch
    h = hierarchy
    m, cfg = _masked_model(h, 4)
    params = parity.calibrated_params(m.net.specs, 11)
    m.load_weights(params)
    b = make_batch(6, cfg["nz"], seed=5)
    m.rng = np.random.RandomState(123)
    preds, recon, latent, edge = m.predict(b["x_g"], b["cond_g"], b["cond2_g"], labels=b["x_g"])
    net = m.net
    x_pad, last = net.x_hat.cpu().numpy().astype(np.float64), float(net.losses[0].cpu())
    o = LM.MaskOracle(h["L"], h["D"], h["U"], h["L_d"], h["D_d"], m.cfg)
    P = {k: torch.from_numpy(v) for k, v in params.items()}
    t = torch.from_numpy
    rng = np.random.RandomState(123)
    eps = np.concatenate([rng.normal(size=(4, cfg["nz"])), rng.normal(size=(4, cfg["nz"]))]).astype(np.float32)
    with torch.no_grad():
        y, y2 = o.cond_embeddings(t(b["cond_g"]), t(b["cond2_g"]), P)
        xh0, _, _ = o.generator(t(b["x_g"][:4]), y[:4], y2[:4], t(eps[:4]), P)
        want0 = float(o.recon_loss(xh0.double() - t(b["x_g"][:4]).double()))
    want = want0 * 4 / 6
    print("predict: masked recon %.6e (oracle %.6e), padded batch %.6e" % (recon, want, last))
    assert abs(recon - want) <= parity.TOL * want
    # the padded batch: rows 2 and 3 are the decoder's output on zero inputs against zero labels
    gt_pad = np.zeros_like(x_pad)
    gt_pad[:2] = b["x_g"][4:]
    assert np.abs(x_pad[:2] - preds[4:]).max() == 0
    want_last = float(o.recon_loss(t(x_pad - gt_pad)))
    assert abs(last - want_last) <= 1e-6 * want_last
    unmasked = float(LM.OO.OptOracle.recon_loss(o, t(x_pad - gt_pad)))
    assert abs(unmasked - want_last) > 1e-4 * want_last              # the mask is what made the difference
    m.rng = np.random.RandomState(123)
    s, r2, _, _ = m.evaluate(b["x_g"], b["cond_g"], b["cond2_g"], labels=b["x_g"])
    assert abs(r2 - recon) <= 1e-6 * recon and "recon loss: {:.2e}".format(r2 * m.lambda_l1) in s


def test_tensorflow_checkpoint_of_a_masked_model(hierarchy, tmp_path):
    """save_tf -> restore through a second masked model: the weights come back unchanged, and the checkpoint holds
    the variables of the unmasked model (the mask is not a variable)."""
    from cape_b200 import tf_checkpoint
    from cape_b200.network import CapeNetwork
    h = hierarchy
    m, cfg = _masked_model(h, 2)
    m.checkpoint_dir = str(tmp_path)
    m.load_weights(parity.calibrated_params(m.net.specs, 9))
    before = m.net.get_params()
    prefix = m.save_tf(3)
    names = {n for n, _, _ in tf_checkpoint.list_variables(prefix)}
    plain = CapeNetwork(h["L"], h["D"], h["U"], h["L_d"], h["D_d"], dict(cfg, loss_mask=None), 1)
    assert {n for n in names if "/Momentum" not in n and n != "global_step"} == set(plain.specs)
    m2, _ = _masked_model(h, 2)
    m2.checkpoint_dir = str(tmp_path)
    assert m2.restore() == prefix
    after = m2.net.get_params()
    assert all(np.array_equal(before[k], after[k]) for k in before)


def test_main_trains_and_tests_with_the_mask(hierarchy, tmp_path, monkeypatch):
    """`python -m cape_b200.main --loss_mask binary`: --mode train on a synthetic dataset writes a checkpoint, and
    --mode test restores it and reports the masked term of the test set (calc_mean: the first batch of four, weighted
    4/6), which differs from the unmasked one."""
    import re
    import test_gpu_smpl as GS
    from cape_b200 import main as M
    cfg_path, _, _, _ = GS._setup(hierarchy, tmp_path)
    data_dir = GS._dataset(tmp_path)
    monkeypatch.chdir(tmp_path)
    losses, _ = M.main(["--config", cfg_path, "--mode", "train", "--loss_mask", "binary", "--num_epochs", "1",
                        "--restart", "1"], project_dir=str(tmp_path))
    assert len(losses) == 1 and np.isfinite(losses[0])
    ck = sorted(f for f in os.listdir(str(tmp_path / "checkpoints" / "e2e")) if f.endswith(".npz"))
    assert ck, os.listdir(str(tmp_path / "checkpoints" / "e2e"))
    out = M.main(["--config", cfg_path, "--mode", "test", "--loss_mask", "binary"], project_dir=str(tmp_path))
    got = float(re.search(r"L1 ([0-9.e+-]+),", out["string"]).group(1))
    # the same evaluation through CAPE with the trained weights, masked and unmasked
    from cape_b200.config_parser import model_params, parse_config
    from cape_b200.models import CAPE
    h = hierarchy
    bd = M.load_body_data(data_dir, "rot")
    recon = {}
    for mask in ("binary", ""):
        args, _ = parse_config(["--config", cfg_path, "--mode", "test", "--loss_mask", mask])
        p = dict(model_params(args), p=h["p"])
        cm = CAPE(L=h["L"], D=h["D"], U=h["U"], L_d=h["L_d"], D_d=h["D_d"], **p)
        cm.build_graph(cm.input_num_verts, cm.nn_input_channel, phase="demo")
        cm.restore()
        cm.rng = np.random.RandomState(args.seed)
        _, recon[mask], _, _ = cm.predict(bd.vertices_test, bd.cond1_test, bd.cond2_test, labels=bd.vertices_test)
    print("main --mode test: reported %.5f, masked %.6f, unmasked %.6f" % (got, recon["binary"], recon[""]))
    assert "{:.5f}".format(recon["binary"]) == "{:.5f}".format(got)
    assert abs(recon["binary"] - recon[""]) > 1e-4 * recon[""]


# =====================================================================================================================
# data parallelism
# =====================================================================================================================
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _dp_worker(rank, world, port, q):
    try:
        root = os.path.dirname(HERE)
        sys.path[:0] = [root, HERE]
        os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1",
                          MASTER_PORT=str(port), NCCL_DEBUG="WARN")
        from cape_b200 import distributed as DP
        from cape_b200 import topology as T
        from cape_b200.network import CapeNetwork
        from cape_b200.params import param_specs
        from cape_b200.synthetic import make_batch
        DP.init("nccl")
        L, D, U, p, L_d, D_d, _ = T.load_graph_mtx(load_for_demo=True)
        cfg = _cfg("affine_l1_mask")
        params = parity.calibrated_params(param_specs(cfg, [l.shape[0] for l in L], [l.shape[0] for l in L_d]), 3)
        N = 2
        order = ("x_g", "cond_g", "cond2_g", "eps", "x_d", "cond_d", "cond2_d")
        full = make_batch(N * world, cfg["nz"], seed=77)
        net = CapeNetwork(L, D, U, L_d, D_d, cfg, N, device=rank, params=params)
        net.set_inputs(*[torch.from_numpy(full[k][rank * N:(rank + 1) * N]) for k in order])
        net.train_step(step=100, allreduce=DP.make_allreduce(world))
        torch.cuda.synchronize()
        out = {"gg": net.PG.grad.cpu().numpy(), "pg": net.PG.flat.cpu().numpy(), "loss": net.losses.cpu().numpy()}
        if rank == 0:
            ref = CapeNetwork(L, D, U, L_d, D_d, cfg, N * world, device=0, params=params)
            ref.set_inputs(*[torch.from_numpy(full[k]) for k in order])
            ref.train_step(step=100)
            torch.cuda.synchronize()
            out.update(ref_gg=ref.PG.grad.cpu().numpy(), ref_pg=ref.PG.flat.cpu().numpy(),
                       ref_loss=ref.losses.cpu().numpy())
        q.put((rank, out))
        import torch.distributed as dist
        dist.barrier()
        dist.destroy_process_group()
    except BaseException as e:          # the parent must not wait for a result that will never come
        import traceback
        q.put((rank, {"error": "".join(traceback.format_exception(type(e), e, e.__traceback__))[-3000:]}))
        os._exit(1)


def test_data_parallel_step_equals_global_batch():
    """Every rank has the same N and the same mask, so the mean of the ranks' masked terms is the global batch's term
    and the averaged gradients are its gradients."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    import torch.multiprocessing as mp
    world, port = 2, _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_dp_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = {}
    try:
        for _ in range(world):
            rank, out = q.get(timeout=240)
            res[rank] = out
            assert "error" not in out, "rank %d failed:\n%s" % (rank, out["error"])
        for p in procs:
            p.join(timeout=60)
            assert p.exitcode == 0
    finally:
        for p in procs:                 # never leave a rank behind
            if p.is_alive():
                p.kill()
    r0, r1 = res[0], res[1]
    assert np.array_equal(r0["gg"], r1["gg"]) and np.array_equal(r0["pg"], r1["pg"])
    recon = 0.5 * (float(r0["loss"][0]) + float(r1["loss"][0]))
    assert abs(recon - float(r0["ref_loss"][0])) <= 1e-6 * float(r0["ref_loss"][0])
    # tolerances of tests/test_gpu_multi.py (the global batch is tiled differently on one GPU)
    e_gg = TP._rel(r0["gg"], r0["ref_gg"])
    e_pg = TP._rel(r0["pg"], r0["ref_pg"])
    print("masked data-parallel vs global batch: generator grads %.2e, parameters %.2e" % (e_gg, e_pg))
    assert e_gg < 3e-4 and e_pg < 1e-6
