"""Pin the oracle: golden known answers, literal numpy transcription, float64 dense polynomials."""
import os

import numpy as np
import pytest
import torch

from oracle import cape_oracle as O
from oracle import np_ops

GOLD = os.path.join(os.path.dirname(__file__), "golden")


def _rel(a, b):
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-30)


def test_golden_ops_numpy(hierarchy):
    from inputs import OPS_VSTRIDE as S, golden_inputs
    g, z = golden_inputs(), np.load(os.path.join(GOLD, "ops_golden.npz"))
    h = hierarchy
    y = np_ops.chebyshev5_np(g["c1_x"], h["L"][0], g["c1_W"], 6)
    assert _rel(y[:, ::S], z["c1_y"]) < 1e-6
    y2 = np_ops.poolwT_np(np_ops.b1leakyrelu_np(np_ops.chebyshev5_np(g["cnp_x"], h["L"][1], g["cnp_W"], 2), g["cnp_b"]),
                          h["D"][1])
    assert _rel(y2[:, ::S], z["cnp_y"]) < 1e-6
    assert _rel(np_ops.poolwT_np(g["up_x"], h["U"][1])[:, ::S], z["up_y"]) < 1e-6


def test_torch_oracle_matches_golden(hierarchy):
    from inputs import OPS_VSTRIDE as S, golden_inputs
    g, z = golden_inputs(), np.load(os.path.join(GOLD, "ops_golden.npz"))
    h = hierarchy
    cfg = dict(F=[64] * 8, K=[2] * 8, Kd=3)
    o = O.Oracle(h["L"], h["D"], h["U"], h["L_d"], h["D_d"], cfg)
    t = torch.from_numpy
    y = o.chebyshev5(t(g["c1_x"]), o.Lt[0], t(g["c1_W"]), 6).numpy()
    assert _rel(y[:, ::S], z["c1_y"]) < 1e-5
    y2 = o.poolwT(o.b1leakyrelu(o.chebyshev5(t(g["cnp_x"]), o.Lt[1], t(g["cnp_W"]), 2), t(g["cnp_b"])), o.Dm[1]).numpy()
    assert _rel(y2[:, ::S], z["cnp_y"]) < 1e-5
    assert _rel(o.poolwT(t(g["up_x"]), o.Um[1]).numpy()[:, ::S], z["up_y"]) < 1e-5


@pytest.mark.parametrize("K", [1, 2, 3, 6])
def test_chebyshev_vs_dense_f64(hierarchy, K):
    """Weight layout W[fin*K + k] and the recurrence against an independent formulation (coarsest level)."""
    L = hierarchy["L_d"][-1]                # 431 vertices: dense T_k is cheap
    rng = np.random.RandomState(K)
    x = rng.normal(size=(3, 431, 5)).astype(np.float32)
    W = rng.normal(0, 0.1, size=(5 * K, 7)).astype(np.float32)
    want = np_ops.chebyshev_dense_f64(x, L, W, K)
    assert _rel(np_ops.chebyshev5_np(x, L, W, K), want) < 1e-5
    o = O.Oracle(hierarchy["L"], hierarchy["D"], hierarchy["U"], hierarchy["L_d"], hierarchy["D_d"],
                 dict(F=[64] * 8, K=[2] * 8, Kd=3), dtype=torch.float64)
    got = o.chebyshev5(torch.from_numpy(x).double(), o.Lt_d[-1], torch.from_numpy(W).double(), K).numpy()
    assert _rel(got, want) < 1e-9


def test_lr_schedule_matches_reference_policy():
    cfg = dict(lr=8e-3, lr_scaler=0.1, decay_steps=10, decay_rate=0.99, lr_warmup=True)
    assert O.lr_schedule(cfg, 0) == (0.0, 0.0)
    g, d = O.lr_schedule(cfg, 40)
    assert abs(g - 8e-3 * 40 / 80) < 1e-12 and abs(d - 8e-4 * 40 / 80) < 1e-12
    g, _ = O.lr_schedule(cfg, 80 + 25)
    assert abs(g - 8e-3 * 0.99 ** 2) < 1e-12
    cfg["lr_warmup"] = False
    assert abs(O.lr_schedule(cfg, 35)[0] - 8e-3 * 0.99 ** 3) < 1e-12


def test_bce_matches_torch():
    l = torch.randn(50, dtype=torch.float64)
    want = torch.nn.functional.binary_cross_entropy_with_logits(l, torch.full_like(l, 0.9))
    assert abs(float(O.Oracle.bce_logits(l, 0.9) - want)) < 1e-12


def test_adam_rule_matches_torch_adam():
    """The oracle's restatement of tf.train.AdamOptimizer against torch.optim.Adam, which differs from TF only in where
    eps enters (eps vs eps * sqrt(1 - b2^t)): identical to 1e-6 for gradients far above eps, three applications."""
    torch.manual_seed(0)
    p0 = torch.randn(1000, dtype=torch.float64)
    p = p0.clone()
    m, v = torch.zeros_like(p), torch.zeros_like(p)
    q = p0.clone().requires_grad_(True)
    opt = torch.optim.Adam([q], lr=3e-3, betas=(O.ADAM_B1, O.ADAM_B2), eps=1e-8)
    for t in (1, 2, 3):
        g = torch.randn(1000, dtype=torch.float64) + 0.5
        p, m, v = O.adam_apply(p, m, v, g, 3e-3, t)
        q.grad = g.clone()
        opt.step()
    assert _rel(p.numpy(), q.detach().numpy()) < 1e-6
    # first application: the step is lr * sign(g) for |g| >> eps
    g = torch.sign(g) * (0.5 + g.abs())
    p1, _, _ = O.adam_apply(p0, torch.zeros_like(p0), torch.zeros_like(p0), g, 3e-3, 1)
    assert _rel((p0 - p1).numpy(), (3e-3 * torch.sign(g)).numpy()) < 1e-6
