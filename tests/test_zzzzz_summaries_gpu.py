"""TensorBoard summaries on the GPU.

- cape_histogram against the float64 transcription of TF's Histogram (tests/summary_oracle.py): single segments of
  1, 3, 31, 4097 and 2^20 + 5 values, and all of nz64's histogrammed variables in one launch; values at +-0, below
  1e-12, float32 neighbours of the bucket limits, denormals, beyond 1e20; non-finite values counted; two calls
  bit-identical;
- cape_loss_ema bit-identical to the float32 host recurrence over 50 applications;
- the summary pass's loss scalars against the CPU oracle (affine nz64 at batch 2, GroupNorm nz18 at batch 1);
- a summary point leaves the training state bit for bit unchanged; CAPE.fit with and without summaries (ref_compat on
  and off) stages the same batches and noise in every application, and its event file has the reference's steps,
  histograms of the saved weights, the learning rates, the validation loss and the moving averages of the
  applications the loop ran;
- `python -m cape_b200.main --mode train` writes summaries/<name>/events.out.tfevents.*.

The file name sorts after every other GPU test file (see tests/test_resblock_encoder_gpu.py for why that matters)."""
import ctypes
import math
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))

import parity  # noqa: E402
import summary_oracle as SO  # noqa: E402

pytestmark = pytest.mark.gpu


def _tp():
    from cape_b200.engine import Topology
    tp = Topology(0)
    tp.reserve_workspace(16 << 20)
    return tp


def _run_histogram(tp, arrays):
    """cape_histogram over float32 arrays (one segment each): (stats [n, 5], nonfinite [n], counts [n, nlim], raw)."""
    from cape_b200 import _lib, summary as S
    dev = [torch.from_numpy(np.ascontiguousarray(a, np.float32).reshape(-1)).cuda() for a in arrays]
    segs = torch.tensor([[t.data_ptr(), t.numel()] for t in dev], dtype=torch.int64).cuda()
    lim = torch.from_numpy(S.bucket_limits()).cuda()
    n, nl = len(dev), lim.numel()
    stats = torch.zeros(n, 5, dtype=torch.float64, device="cuda")
    nonfinite = torch.zeros(n, dtype=torch.int64, device="cuda")
    counts = torch.zeros(n, nl, dtype=torch.int64, device="cuda")
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    _lib.check(tp.lib.cape_histogram(tp.h, p(segs), n, p(lim), nl, p(stats), p(nonfinite), p(counts),
                                     ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    return stats.cpu().numpy(), nonfinite.cpu().numpy(), counts.cpu().numpy()


def _edge_values(n, rng):
    from cape_b200 import summary as S
    lim = S.bucket_limits()
    inner = lim[(np.abs(lim) > 0) & (np.abs(lim) < 1e20)].astype(np.float32)
    near = np.concatenate([inner, np.nextafter(inner, np.float32(np.inf)), np.nextafter(inner, np.float32(-np.inf))])
    special = np.float32([0.0, -0.0, 5e-13, -5e-13, 1e-30, 1e-45, -1e-45, 1e-39, -2e-40, 2e20, -5e25, 3.4e38, -3.4e38])
    pool = np.concatenate([near, special, rng.normal(0, 0.1, 4096).astype(np.float32)])
    return pool[rng.randint(0, pool.size, size=n)]


def _check(stats, counts, values):
    mn, mx, num, sm, sq, want = SO.histogram(values)
    x = np.asarray(values, np.float32).astype(np.float64)
    assert np.array_equal(counts, want)
    assert stats[2] == num
    # exact, sign of zero included
    assert np.float64(stats[0]).tobytes() == np.float64(mn).tobytes(), (stats[0], mn)
    assert np.float64(stats[1]).tobytes() == np.float64(mx).tobytes(), (stats[1], mx)
    assert abs(stats[3] - sm) <= 1e-12 * math.fsum(np.abs(x)), (stats[3], sm)
    assert abs(stats[4] - sq) <= 1e-12 * sq, (stats[4], sq)


@pytest.mark.parametrize("n", [1, 3, 31, 4097, (1 << 20) + 5])
def test_histogram_single_segment(n):
    rng = np.random.RandomState(n % 1000)
    v = _edge_values(n, rng)
    if n == 3:
        v = np.float32([-0.0, 0.0, -0.0])            # min and max are the first zero: -0.0
    stats, nonfinite, counts = _run_histogram(_tp(), [v])
    assert nonfinite[0] == 0
    _check(stats[0], counts[0], v)


def test_histogram_all_nz64_variables_in_one_launch(hierarchy):
    from cape_b200 import summary as S
    from cape_b200.params import NZ64_AFFINE, param_specs
    h = hierarchy
    specs = param_specs(dict(NZ64_AFFINE), [l.shape[0] for l in h["L"]], [l.shape[0] for l in h["L_d"]])
    names = S.histogram_names(specs)
    params = parity.calibrated_params(specs, 5)
    rng = np.random.RandomState(9)
    arrays = []
    for i, n in enumerate(names):
        a = np.asarray(params[n], np.float32).reshape(-1).copy()
        if i % 3 == 0:                                 # sprinkle edge values into every third variable
            k = max(1, a.size // 50)
            a[rng.randint(0, a.size, size=k)] = _edge_values(k, rng)
        arrays.append(a)
    assert len(arrays) == 45 and 2.1e6 < sum(a.size for a in arrays) < 2.3e6
    tp = _tp()
    stats, nonfinite, counts = _run_histogram(tp, arrays)
    assert not nonfinite.any()
    for i, a in enumerate(arrays):
        _check(stats[i], counts[i], a)
    again = _run_histogram(tp, arrays)
    assert stats.tobytes() == again[0].tobytes() and counts.tobytes() == again[2].tobytes()


def test_histogram_counts_non_finite_values():
    rng = np.random.RandomState(4)
    a = rng.normal(size=10000).astype(np.float32)
    bad = rng.choice(a.size, 7, replace=False)
    a[bad[:3]], a[bad[3:5]], a[bad[5:]] = np.nan, np.inf, -np.inf
    b = rng.normal(size=100).astype(np.float32)
    stats, nonfinite, counts = _run_histogram(_tp(), [a, b])
    assert nonfinite.tolist() == [7, 0]
    fin = np.delete(a, bad)
    _check(stats[0], counts[0], fin)
    _check(stats[1], counts[1], b)


def test_loss_ema_is_the_float32_recurrence():
    """50 applications: random loss buffers and FC kernels, all four lambdas and the regularisation non-zero; the
    device shadows equal the host float32 recurrence bit for bit after every application."""
    from cape_b200 import _lib
    from cape_b200.engine import Topology
    tp = Topology(0)
    cfg = dict(lambda_gan=0.1, lambda_recon=1.3, lambda_edge=0.7, lambda_latent=8e-4, regularization=2e-3)
    rng = np.random.RandomState(8)
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    st = lambda: ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    shadow = torch.zeros(2, device="cuda")
    fc = torch.zeros(1, device="cuda")
    apps = []
    for it in range(50):
        losses = torch.from_numpy(np.abs(rng.normal(size=8)).astype(np.float32) * 3).cuda()
        Ws = [torch.from_numpy(rng.normal(0, 0.05, size=n).astype(np.float32)).cuda() for n in (1000, 1000, 4003)]
        fc.zero_()
        for W in Ws:
            _lib.check(tp.lib.cape_sumsq(p(W), W.numel(), p(fc), st()))
        _lib.check(tp.lib.cape_loss_ema(p(losses), p(fc), cfg["lambda_gan"], cfg["lambda_recon"], cfg["lambda_edge"],
                                        cfg["lambda_latent"], cfg["regularization"], 0.9, p(shadow), st()))
        torch.cuda.synchronize()
        apps.append((losses.cpu().numpy(), fc.cpu().numpy()[0]))
        want = SO.loss_average(apps, cfg)
        got = shadow.cpu().numpy()
        assert got[0] == want[0] and got[1] == want[1], (it, got, want)
    assert np.all(np.isfinite(got)) and got[0] > 0


@pytest.mark.parametrize("which", ["nz64", "nz18"])
def test_summary_pass_against_the_oracle(hierarchy, which):
    """enqueue_loss_forward + the FC sum of squares: the five loss scalars and fc_regularization_g within 1e-4 of the
    oracle's forward on the same weights, batch and noise."""
    from cape_b200.network import CapeNetwork
    from cape_b200.params import NZ18_PLAIN, NZ64_AFFINE, param_specs
    from cape_b200.synthetic import make_batch
    from cape_b200 import summary as S
    h = hierarchy
    cfg, N = (dict(NZ64_AFFINE, decay_steps=10), 2) if which == "nz64" else (dict(NZ18_PLAIN, decay_steps=10), 1)
    specs = param_specs(cfg, [l.shape[0] for l in h["L"]], [l.shape[0] for l in h["L_d"]])
    params = parity.calibrated_params(specs, 123, 0.05)
    net = CapeNetwork(h["L"], h["D"], h["U"], h["L_d"], h["D_d"], cfg, N, params=params)
    tb = {k: torch.from_numpy(v) for k, v in make_batch(N, cfg["nz"], seed=77).items()}
    net.set_inputs(tb["x_g"], tb["cond_g"], tb["cond2_g"], tb["eps"], tb["x_d"], tb["cond_d"], tb["cond2_d"])
    net.track_loss_average()
    net.enqueue_loss_forward()
    net.enqueue_fc_sumsq()
    torch.cuda.synchronize()
    got = net.loss_dict()
    r = np.float32(cfg["regularization"])
    reg = r * (r * (net.fc_sumsq.cpu().numpy()[0] * np.float32(0.5)))
    o_params = {k: np.asarray(v, np.float32) for k, v in params.items()}
    res, _, _ = parity._oracle_update(h, cfg, o_params, {k: np.zeros_like(v) for k, v in o_params.items()}, tb, 100,
                                      torch.float32, False)
    for k in ("recon", "edge", "latent", "gan_g", "gan_d"):
        assert abs(got[k] - res[k]) <= 1e-4 * max(abs(res[k]), 1e-30), (k, got[k], res[k])
    want_reg = cfg["regularization"] ** 2 * sum(float((o_params[n].astype(np.float64) ** 2).sum())
                                                for n in S.FC_REGULARISED) / 2
    assert abs(reg - want_reg) <= 1e-4 * want_reg


def _cape(h, ref_compat, tmp_path, summaries):
    from cape_b200.config_parser import model_params, parse_config
    from cape_b200.models import CAPE
    tmp_path.mkdir(parents=True, exist_ok=True)
    fn = tmp_path / "c.yaml"
    fn.write_text("nz: 64\nnz_cond: 32\nnz_cond2: 32\naffine: 1\nlr_warmup: 1\nname: sum_test\nbatch_size: 2\n"
                  "mode: demo\nregularization: 0.002\n")
    args, _ = parse_config(["--config", str(fn)])
    p = dict(model_params(args), p=h["p"], ref_compat=ref_compat, restart=True, num_epochs=2,
             checkpoint_dir=str(tmp_path / ("ck_on" if summaries else "ck_off")),
             summary_dir=str(tmp_path / "summaries") if summaries else None)
    m = CAPE(L=h["L"], D=h["D"], U=h["U"], L_d=h["L_d"], D_d=h["D_d"], **p)
    m.build_graph(m.input_num_verts, m.nn_input_channel, phase="train")
    m.load_weights(parity.calibrated_params(m.net.specs, 31))
    return m


@pytest.mark.parametrize("ref_compat", [True, False])
def test_fit_with_and_without_summaries(hierarchy, tmp_path, ref_compat):
    """Summaries change nothing of the training: every application stages the same batch and noise with summaries on
    and off, and global_step agrees.  The training step itself is not bit-reproducible from run to run (the bias /
    condition column sums accumulate with float atomics, and eight GAN updates amplify that to 2e-1 relative in some
    tensors, also between two runs without summaries), so the weights are printed, not asserted;
    test_summary_pass_leaves_the_training_state_alone checks bit for bit that a summary point changes no training
    state."""
    import test_gpu_api as GA
    from cape_b200 import summary as S
    h = hierarchy
    data = GA._synthetic_data(4, 3, seed=3)            # 3 validation meshes: calc_mean gives the first batch weight 2/3
    runs = {}
    for key, on in (("off", False), ("on", True), ("off2", False)):
        m = _cape(h, ref_compat, tmp_path / key, on)
        net, apps, staged = m.net, [], []
        orig = net.train_step

        def spy(step=None, **kw):
            staged.append(b"".join(t.cpu().numpy().tobytes() for t in (net.in_x, net.in_cond, net.in_cond2, net.in_eps,
                                                                       net.xcat[:net.N])) + bytes([step % 256]))
            r = orig(step=step, **kw)
            if net.loss_avg is not None:
                apps.append((net.losses.cpu().numpy().copy(), net.fc_sumsq.cpu().numpy()[0]))
            return r

        net.train_step = spy
        np.random.seed(17)
        losses, _ = m.fit(data)
        net.train_step = orig
        runs[key] = (m, losses, apps, staged)
    m1, l1, apps, st1 = runs["on"][:4]
    steps = [2, 4]                                     # 4 training meshes / batch 2: two loop steps per epoch
    per_step = 2 if ref_compat else 1
    assert len(apps) == 4 * per_step
    assert st1 == runs["off"][3] == runs["off2"][3]
    assert all(len(runs[k][1]) == 2 and all(np.isfinite(runs[k][1])) for k in runs)
    ck = lambda key, s: np.load(str(tmp_path / key / ("ck_on" if key == "on" else "ck_off") / "sum_test"
                                    / ("model-%d.npz" % s)))
    spread, worst = 0.0, 0.0
    for s in steps:
        a, b, c = ck("off", s), ck("on", s), ck("off2", s)
        assert sorted(a.files) == sorted(b.files)
        assert int(a["global_step"]) == int(b["global_step"])
        for k in a.files:
            if k != "global_step":
                worst = max(worst, parity.rel(b[k], a[k]))
                spread = max(spread, parity.rel(c[k], a[k]))
    print("summaries on vs off: max rel %.2e; two runs without summaries: %.2e" % (worst, spread))
    summ = tmp_path / "on" / "summaries" / "sum_test"
    files = S.event_files(str(summ))
    assert len(files) == 1
    ev = SO.read_events(files[0])
    assert ev[0]["file_version"] == "brain.Event:2"
    assert [e["step"] for e in ev[1:]] == steps
    names = m1.net.histogram_names()
    for i, (e, s) in enumerate(zip(ev[1:], steps)):
        assert e["tags"] == list(S.SCALAR_TAGS) + [S.VALIDATION_TAG] + names
        sc = e["scalars"]
        assert sc[S.VALIDATION_TAG] == np.float32(l1[i])
        w = ck("on", s)
        gs = int(w["global_step"])
        lr_g, lr_d = m1.net.lr_now(gs)
        assert sc["training/lr_g"] == np.float32(lr_g) and sc["training/lr_d"] == np.float32(lr_d)
        avg = SO.loss_average(apps[: s * per_step], m1.cfg)
        assert sc["loss/averages/loss_g"] == avg[0] and sc["loss/averages/loss_d"] == avg[1]
        assert sc["loss/fc_regularization_d"] == 0.0
        assert all(np.isfinite(v) for v in sc.values())
        for n in names:
            mn, mx, num, sm, sq, counts = SO.histogram(w[n])
            lim, cnt = SO.collapse(S.bucket_limits(), counts)
            got = e["histograms"][n]
            assert (got["min"], got["max"], got["num"]) == (mn, mx, num), n
            assert got["bucket_limit"] == lim and got["bucket"] == cnt, n
            assert abs(got["sum"] - sm) <= 1e-12 * math.fsum(np.abs(w[n].astype(np.float64)).ravel()), n
            assert abs(got["sum_squares"] - sq) <= 1e-12 * sq, n


def test_summary_pass_leaves_the_training_state_alone(hierarchy, tmp_path):
    """After an update, the summary point (forward pass, FC sum of squares, histograms, encoding) leaves the weights,
    gradients, momentum, derived weight layouts, step counters and the moving averages bit for bit as they were."""
    from cape_b200.synthetic import make_batch
    m = _cape(hierarchy, False, tmp_path, True)
    net = m.net
    m._open_summaries().close()
    tb = {k: torch.from_numpy(v) for k, v in make_batch(2, 64, seed=5).items()}
    net.set_inputs(tb["x_g"], tb["cond_g"], tb["cond2_g"], tb["eps"], tb["x_d"], tb["cond_d"], tb["cond2_d"])
    net.train_step(step=0)
    torch.cuda.synchronize()
    bufs = lambda: [b.detach().cpu().numpy().tobytes() for b in
                    (net.PG.flat, net.PD.flat, net.PG.grad, net.PD.grad, net.PG.mom, net.PD.mom, net.loss_avg)
                    + tuple(l.Wt for l in net.all_layers())]
    before, counters = bufs(), (net.step_count, net.adam_t)
    scalars, histograms = m._summary_values()
    torch.cuda.synchronize()
    assert bufs() == before and (net.step_count, net.adam_t) == counters
    assert len(histograms) == len(net.histogram_names()) and len(scalars) == 10


def test_restart_removes_only_event_files(hierarchy, tmp_path):
    import test_gpu_api as GA
    from cape_b200 import summary as S
    d = tmp_path / "summaries" / "sum_test"
    d.mkdir(parents=True)
    (d / "events.out.tfevents.0000000001.old").write_bytes(b"")
    (d / "keep.txt").write_text("x")
    m = _cape(hierarchy, False, tmp_path, True)
    m.num_epochs = 1
    np.random.seed(1)
    m.fit(GA._synthetic_data(4, 2, seed=3))
    files = S.event_files(str(d))
    assert len(files) == 1 and not files[0].endswith(".old")
    assert (d / "keep.txt").read_text() == "x"


def test_main_train_writes_summaries(hierarchy, tmp_path, monkeypatch):
    """`python -m cape_b200.main --mode train` writes summaries/<name>/events.out.tfevents.* in the working directory,
    readable by TensorBoard's loader when it is installed."""
    import test_gpu_smpl as GS
    from cape_b200 import main as M
    from cape_b200 import summary as S
    cfg_path, _, _, _ = GS._setup(hierarchy, tmp_path)
    GS._dataset(tmp_path)
    monkeypatch.chdir(tmp_path)
    losses, _ = M.main(["--config", cfg_path, "--mode", "train", "--num_epochs", "1", "--restart", "1"],
                       project_dir=str(tmp_path))
    files = S.event_files(str(tmp_path / "summaries" / "e2e"))
    assert len(files) == 1
    ev = SO.read_events(files[0])
    assert len(ev) == 2 and ev[1]["scalars"][S.VALIDATION_TAG] == np.float32(losses[0])
    assert set(S.SCALAR_TAGS) <= set(ev[1]["scalars"])
    try:
        from tensorboard.backend.event_processing import event_file_loader as EFL
    except ImportError:
        return
    tags = {v.tag for e in EFL.EventFileLoader(files[0]).Load() for v in e.summary.value}
    assert set(S.SCALAR_TAGS) | {S.VALIDATION_TAG} <= tags
