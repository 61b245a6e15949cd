"""Parity checks of the CUDA path (through the C ABI) against the CPU oracle.  Each function returns a dict
{name: relative error}; tests assert on them, tests/gpu_check.py prints them all."""
import os

import numpy as np
import torch

from oracle import cape_oracle as O
from oracle import np_ops

GOLD = os.path.join(os.path.dirname(__file__), "golden")
TOL = 1e-4   # BASELINE.json north_star: 1e-4 relative fp32


def rel(a, b):
    a = np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def vertex_l2(a, b):
    """max_v ||a_v - b_v||_2 / max_v ||b_v||_2 (BASELINE.md section 4)."""
    a = np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b, axis=-1).max() / max(np.linalg.norm(b, axis=-1).max(), 1e-30))


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def golden_ops(h):
    from inputs import OPS_VSTRIDE as S, golden_inputs
    from cape_b200 import ops
    g, z = golden_inputs(), np.load(os.path.join(GOLD, "ops_golden.npz"))
    out = {}
    y = ops.chebyshev5(_cuda(g["c1_x"]), h["L"][0], _cuda(g["c1_W"]), 6)
    out["C1 cheb K=6 [1,6890,3]->64 (max-rel)"] = rel(y.cpu().numpy()[:, ::S], z["c1_y"])
    out["C1 cheb K=6 (vertex-L2)"] = vertex_l2(y.cpu().numpy()[:, ::S], z["c1_y"])
    y = ops.chebyshev5(_cuda(g["cnp_x"]), h["L"][1], _cuda(g["cnp_W"]), 2, bias=_cuda(g["cnp_b"]),
                       activation="b1leakyrelu", pool=h["D"][1])
    out["cnp K=2 16->32 +bias+leaky+pool"] = rel(y.cpu().numpy()[:, ::S], z["cnp_y"])
    y = ops.poolwT(_cuda(g["up_x"]), h["U"][1])
    out["unpool 3445->6890"] = rel(y.cpu().numpy()[:, ::S], z["up_y"])
    return out


def cheb_grads(tag, L, K, Fin, Fout, N, U=None, D=None, act="b1leakyrelu", seed=0):
    """forward + all gradients of chebyshev5 (+ fused unpool U / bias+act / pool D) vs oracle autograd."""
    from cape_b200 import ops
    rng = np.random.RandomState(seed)
    Min = U.shape[1] if U is not None else L.shape[0]
    x = rng.normal(size=(N, Min, Fin)).astype(np.float32)
    W = rng.normal(0, 0.1, size=(Fin * K, Fout)).astype(np.float32)
    b = rng.normal(0, 0.1, size=(1, L.shape[0], Fout) if act == "b2relu" else (Fout,)).astype(np.float32)
    o = O.Oracle([L], [D] if D is not None else [], [U] if U is not None else [], [], [], dict(F=[Fout], K=[K], Kd=3))
    xt, Wt, bt = (torch.from_numpy(a).requires_grad_(True) for a in (x, W, b))
    z = xt
    if U is not None:
        z = o.poolwT(z, o.Um[0])
    z = o.chebyshev5(z, o.Lt[0], Wt, K)
    if act is not None:
        z = getattr(o, act)(z, bt)                    # b1leakyrelu | b1relu | b2relu | b1tanh, models.py:105-127
    if D is not None:
        z = o.poolwT(z, o.Dm[0])
    dy = rng.normal(size=tuple(z.shape)).astype(np.float32)
    z.backward(torch.from_numpy(dy))
    xc, Wc, bc = (_cuda(a).requires_grad_(True) for a in (x, W, b))
    y = ops.chebyshev5(xc, L, Wc, K, bias=bc if act else None, activation=act, pool=D, unpool=U)
    y.backward(_cuda(dy))
    out = {tag + " fwd": rel(y.detach().cpu().numpy(), z.detach().numpy()),
           tag + " dx": rel(xc.grad.cpu().numpy(), xt.grad.numpy()),
           tag + " dW": rel(Wc.grad.cpu().numpy(), Wt.grad.numpy())}
    if act:
        out[tag + " db"] = rel(bc.grad.cpu().numpy(), bt.grad.numpy())
    return out


def cheb_grad_cases(h):
    out = {}
    out.update(cheb_grads("enc-like L1 K=2 64->64 +pool", h["L"][1], 2, 64, 64, 2, D=h["D"][1]))
    out.update(cheb_grads("dec-like L5 K=2 40->24 +unpool", h["L"][5], 2, 40, 24, 3, U=h["U"][5], act=None))
    out.update(cheb_grads("disc-like Ld1 K=3 64->64 +pool", h["L_d"][1], 3, 64, 64, 2, D=h["D_d"][1]))
    out.update(cheb_grads("1x1 L8 K=1 512->64", h["L"][8], 1, 512, 64, 2, act=None))
    out.update(cheb_grads("thin L0 K=2 32->3", h["L"][0], 2, 32, 3, 2, act=None))
    out.update(cheb_grads("first L0 K=2 3->64", h["L"][0], 2, 3, 64, 2))
    out.update(cheb_grads("odd Ld4 K=2 13->1 relu", h["L_d"][4], 2, 13, 1, 5, act="b1relu"))
    # wide same-level layer through the plain op API (no pre-split weight copies), more 128-row tiles than SMs:
    # persistent kernel, identity term by TMA, weights by the producer warps
    out.update(cheb_grads("wide L6 K=2 128->256 multi-tile", h["L"][6], 2, 128, 256, 24, act=None))
    # the rest of base_model's operator seam (unused by the shipped configs): udn = unpool + conv + bias/act in one
    # launch, per-vertex bias (b2relu), tanh (its gradient is smooth: no imposed decisions needed)
    out.update(cheb_grads("udn L5 K=2 64->32 +unpool b1tanh", h["L"][5], 2, 64, 32, 2, U=h["U"][5], act="b1tanh"))
    out.update(cheb_grads("b2relu L8 K=2 32->16 per-vertex bias", h["L"][8], 2, 32, 16, 1, act="b2relu"))
    return out


def plain_operand_cases(h):
    """Calls whose terms are all plain tensors (1x1 convs) take the plain-operand tensor-core path: widths that are not
    multiples of the column tile or exceed one tile (GroupNorm blocks: 544, 288, 160), multi-tile row counts, and the
    precise (split accumulation chains) mode; forward, dX, dW against the oracle."""
    out = {}
    out.update(cheb_grads("plain L8 K=1 512->64", h["L"][8], 1, 512, 64, 4, act=None))
    out.update(cheb_grads("plain L8 K=1 256->544", h["L"][8], 1, 256, 544, 3, act=None))
    r = cheb_grads("plain L6 K=1 160->288 leaky", h["L"][6], 1, 160, 288, 2, seed=3)
    out.update({k: v for k, v in r.items() if k.endswith(" fwd")})      # no imposed decisions here: forward only
    out.update(cheb_grads("plain L6 K=1 160->288", h["L"][6], 1, 160, 288, 2, act=None, seed=3))
    out.update(cheb_grads("plain L4 K=1 96->32 multi-tile", h["L"][4], 1, 96, 32, 30, act=None, seed=4))
    return out


def precise_vs_truth(h):
    """cape_conv_args.precise against a float64 truth: the plain-operand kernel with split accumulation chains must be
    markedly closer to it than the default single-chain accumulation (entries: precise error / default error)."""
    from cape_b200 import ops
    o = O.Oracle(h["L"], h["D"], h["U"], h["L_d"], h["D_d"], dict(F=[64] * 8, K=[2] * 8, Kd=3), dtype=torch.float64)
    g = torch.Generator(device="cuda").manual_seed(2)
    out = {}
    for tag, lvl, Fin, Fout, N in (("L8 1024->512", 8, 1024, 512, 8), ("L8 512->64", 8, 512, 64, 8)):
        x = torch.randn(N, h["L"][lvl].shape[0], Fin, device="cuda", generator=g)
        x = torch.where(x > 0, x, 0.2 * x)
        W = torch.randn(Fin, Fout, device="cuda", generator=g) * 0.1
        want = o.chebyshev5(x.cpu().double(), o.Lt[lvl], W.cpu().double(), 1).numpy()
        e = {}
        for precise in (False, True):
            y = ops.chebyshev5(x, h["L"][lvl], W, 1, precise=precise).cpu().numpy()
            e[precise] = rel(y, want)
        out["precise %s (max-rel vs fp64)" % tag] = e[True]
        out["default %s (max-rel vs fp64)" % tag] = e[False]
    return out


def apply_cases(h):
    """cape_apply (operators without contraction) against scipy: composed conv operators, transposes, scaled two-term
    recurrence steps, strided outputs, the condition term and every epilogue."""
    import scipy.sparse as sp
    from cape_b200 import engine as E
    from cape_b200 import ops
    from cape_b200 import topology as T
    tp = ops.topology_for(torch.device("cuda", 0))
    rng = np.random.RandomState(0)
    out = {}

    def dense_apply(m, x):
        m = sp.csr_matrix(m).astype(np.float64)
        return np.stack([m @ x[n].astype(np.float64) for n in range(x.shape[0])])

    # (1) un-pooling conv operators on 128-wide rows, two accumulators, condition term, AFFINE epilogue
    site = E.ConvSite(tp, h["L"][5], 2, U=h["U"][5])
    N, Fo, C = 3, 128, 8
    z = rng.normal(size=(N, site.rows_in, 3 * Fo)).astype(np.float32)
    y = rng.normal(size=(N, C)).astype(np.float32)
    wc = rng.normal(size=(3, C, Fo)).astype(np.float32)
    zc, yc, wcc = _cuda(z), _cuda(y), _cuda(wc)
    o1, o2 = torch.empty(N, site.rows_out, Fo, device="cuda"), torch.empty(N, site.rows_out, Fo, device="cuda")
    terms = [dict(src=zc[:, :, k * Fo:], op=site.ops[k], src_rows=site.rows_in, src_stride=3 * Fo, acc=0, wc=wcc[k],
                  wc_stride=Fo) for k in range(2)]
    terms.append(dict(src=zc[:, :, 2 * Fo:], op=site.ops[0], src_rows=site.rows_in, src_stride=3 * Fo, acc=1, wc=wcc[2],
                      wc_stride=Fo))
    E.apply_call(tp, N, site.rows_out, Fo, terms, o1, out2=o2, cond=yc, epilogue=E.EPI_AFFINE)
    rs = [np.asarray(m.sum(1)).reshape(1, -1, 1) for m in site.mats]
    q = np.einsum("nc,kcf->knf", y.astype(np.float64), wc.astype(np.float64))[:, :, None, :]
    acc0 = sum(dense_apply(site.mats[k], z[:, :, k * Fo:(k + 1) * Fo]) + rs[k] * q[k] for k in range(2))
    acc1 = dense_apply(site.mats[0], z[:, :, 2 * Fo:]) + rs[0] * q[2]
    out["apply unpool affine out"] = rel(o1.cpu().numpy(), acc1 + np.maximum(acc0, 0))
    out["apply unpool affine out2"] = rel(o2.cpu().numpy(), np.maximum(acc0, 0))
    # (2) transposed pooled K=3 operators on 64-wide rows, SLOPE epilogue
    site = E.ConvSite(tp, h["L_d"][1], 3, D=h["D_d"][1])
    N, F = 2, 64
    z = rng.normal(size=(N, site.rows_out, 3 * F)).astype(np.float32)
    aux = rng.normal(size=(N, site.rows_in, F)).astype(np.float32)
    o1 = torch.empty(N, site.rows_in, F, device="cuda")
    zc = _cuda(z)
    E.apply_call(tp, N, site.rows_in, F, [dict(src=zc[:, :, k * F:], op=site.opsT[k], src_rows=site.rows_out,
                                               src_stride=3 * F) for k in range(3)], o1, epilogue=E.EPI_SLOPE,
                 aux=_cuda(aux), alpha=0.2)
    want = sum(dense_apply(site.mats[k].T, z[:, :, k * F:(k + 1) * F]) for k in range(3)) * np.where(aux > 0, 1.0, 0.2)
    out["apply pooled^T K=3 slope"] = rel(o1.cpu().numpy(), want)
    # (3) one step of the recurrence, T_2 x = 2 L~ (L~ x) - x, odd width, strided output, bias + leaky
    L = h["L"][3]
    Lt = T.rescale_L(L)
    op = tp.add_operator(Lt)
    N, F = 2, 36
    x = rng.normal(size=(N, L.shape[0], F)).astype(np.float32)
    b = rng.normal(size=(F,)).astype(np.float32)
    xc = _cuda(x)
    b1 = torch.empty(N, L.shape[0], F, device="cuda")
    E.apply_call(tp, N, L.shape[0], F, [dict(src=xc, op=op, src_rows=L.shape[0], src_stride=F)], b1)
    wide = torch.zeros(N, L.shape[0], 2 * F, device="cuda")
    E.apply_call(tp, N, L.shape[0], F, [dict(src=b1, op=op, src_rows=L.shape[0], src_stride=F, scale=2.0),
                                        dict(src=xc, op=-1, src_rows=L.shape[0], src_stride=F, scale=-1.0)],
                 wide[:, :, F:], out_stride=2 * F, bias=_cuda(b), act=E.ACT_LEAKY)
    t2 = 2 * dense_apply(Lt, dense_apply(Lt, x)) - x + b
    out["apply recurrence T2 (strided, bias, leaky)"] = rel(wide[:, :, F:].cpu().numpy(), np.where(t2 > 0, t2, 0.2 * t2))
    out["apply strided output leaves the rest"] = float(wide[:, :, :F].abs().max())
    # (4) separate outputs: the three basis tensors of a pooled K=3 layer in one launch
    site = E.ConvSite(tp, h["L_d"][2], 3, D=h["D_d"][2])
    N, F = 3, 64
    x = rng.normal(size=(N, site.rows_in, F)).astype(np.float32)
    xc = _cuda(x)
    B = torch.empty(3, N, site.rows_out, F, device="cuda")
    E.apply_call(tp, N, site.rows_out, F, [dict(src=xc, op=site.ops[k], src_rows=site.rows_in, src_stride=F) for k in range(3)],
                 B, term_stride=B.stride(0))
    for k in range(3):
        out["apply separate outputs term %d" % k] = rel(B[k].cpu().numpy(), dense_apply(site.mats[k], x))
    return out


def gemm_cases():
    from cape_b200 import ops
    from cape_b200.engine import gemm, ACT_LEAKY
    tp = ops.topology_for(torch.device("cuda", 0))
    rng = np.random.RandomState(1)
    out = {}
    for (M, N, K, ta, tb, bias, act) in [(64, 128, 55168, False, False, True, 0), (64, 5000, 128, False, True, False, 0),
                                         (300, 130, 64, True, False, False, 0), (7, 3, 2, False, False, True, 1),
                                         (1, 20670, 5, False, False, False, 0), (33, 64, 1, True, True, False, 0),
                                         # the four operand layouts of the vectorised kernel (FC forward / dW / dx shapes)
                                         (5000, 64, 64, True, False, True, 1), (4100, 64, 64, True, True, False, 0),
                                         (64, 4100, 64, False, True, False, 0), (1, 55168, 64, False, False, False, 0)]:
        A = rng.normal(size=(K, M) if ta else (M, K)).astype(np.float32)
        B = rng.normal(size=(N, K) if tb else (K, N)).astype(np.float32)
        bv = rng.normal(size=(N,)).astype(np.float32) if bias else None
        C0 = rng.normal(size=(M, N)).astype(np.float32)
        Am, Bm = (A.T if ta else A), (B.T if tb else B)
        want = 0.5 * (Am.astype(np.float64) @ Bm.astype(np.float64))
        if bias:
            want = want + bv
        if act:
            want = np.where(want > 0, want, 0.2 * want)
        want = want + 2.0 * C0
        Ac, Bc, Cc = _cuda(A), _cuda(B), _cuda(C0)
        gemm(tp, Ac.t() if ta else Ac, Bc.t() if tb else Bc, Cc, bias=_cuda(bv) if bias else None,
             act=ACT_LEAKY if act else 0, alpha=0.5, beta=2.0)
        out["gemm M%d N%d K%d ta%d tb%d" % (M, N, K, ta, tb)] = rel(Cc.cpu().numpy(), want)
    return out


def gn_case(N=2, rows=862, C=544, seed=0):
    from cape_b200 import ops, _lib
    from cape_b200 import engine as E
    tp = ops.topology_for(torch.device("cuda", 0))
    rng = np.random.RandomState(seed)
    x = (rng.normal(size=(N, rows, C)) * 1.5 + 0.3).astype(np.float32)
    gm = rng.normal(1, 0.2, size=(C,)).astype(np.float32)
    bt = rng.normal(0, 0.2, size=(C,)).astype(np.float32)
    dy = rng.normal(size=(N, rows, C)).astype(np.float32)
    o = O.Oracle([], [], [], [], [], dict(F=[C], K=[2], Kd=3))
    xt, gt, btt = (torch.from_numpy(a).double().requires_grad_(True) for a in (x, gm, bt))
    yt = torch.relu(o.gn(xt, gt, btt))
    yt.backward(torch.from_numpy(dy).double())
    G = min(32, C)
    xc, gc, bc, dyc = _cuda(x), _cuda(gm), _cuda(bt), _cuda(dy)
    y = torch.empty_like(xc)
    stats = torch.empty(N, G, 2, device="cuda")
    _lib.check(tp.lib.cape_gn_relu_fwd(tp.h, E._ptr(xc), N, rows, C, G, 1e-5, E._ptr(gc), E._ptr(bc), E._ptr(y),
                                       E._ptr(stats), E._stream()))
    dx = torch.empty_like(xc)
    dg, db = torch.zeros(C, device="cuda"), torch.zeros(C, device="cuda")
    _lib.check(tp.lib.cape_gn_relu_bwd(tp.h, E._ptr(xc), E._ptr(y), E._ptr(dyc), N, rows, C, G, E._ptr(gc),
                                       E._ptr(stats), E._ptr(dx), 0, E._ptr(dg), E._ptr(db), E._stream()))
    t = "gn C=%d rows=%d " % (C, rows)
    return {t + "fwd": rel(y.cpu().numpy(), yt.detach().numpy()), t + "dx": rel(dx.cpu().numpy(), xt.grad.numpy()),
            t + "dgamma": rel(dg.cpu().numpy(), gt.grad.numpy()), t + "dbeta": rel(db.cpu().numpy(), btt.grad.numpy())}


def calibrated_params(specs, seed=123, fc_scale=0.05):
    """Reference initialisers, with the encoder's fc_mean / fc_var kernels scaled down so that the KL term is O(1)
    as in a trained model.  With raw glorot init on N(0,1) inputs logvar reaches +-10, exp(logvar) ~ 1e4, the KL
    term is ~1e4 and single leaky-ReLU sign flips (fp32 rounding) move conv gradients by 1e-3: ill-conditioned for
    ANY fp32 implementation, so not a meaningful parity regime (both regimes are reported by tests/gpu_check.py)."""
    from cape_b200.params import init_params
    params = init_params(specs, seed)
    for k in params:
        if k.endswith("fc_mean/dense/kernel") or k.endswith("fc_var/dense/kernel"):
            params[k] = (params[k] * fc_scale).astype(np.float32)
    return params


def cuda_masks(net, h, N):
    """Branch decisions (activation > 0) of every (leaky-)ReLU site taken from the CUDA forward, in the reference's
    vertex numbering, keyed like Oracle.masks; pooled sites only know the selected rows (second dict)."""
    import scipy.sparse as sp
    from cape_b200 import topology as T2
    masks, rows = {}, {}

    def sel(D):
        return None if T2.is_identity(D, tol=0) else torch.from_numpy(sp.csr_matrix(D).indices.astype(np.int64))

    def pos(a, order):
        m = (a > 0).cpu()
        return m if order is None else m[:, torch.from_numpy(T2.inverse_order(order))]

    for i, a in enumerate(net.enc_act):
        masks["enc%d" % (i + 1)] = pos(a, net.enc[i].site.order_out)
        r = sel(h["D"][i])
        if r is not None:
            rows["enc%d" % (i + 1)] = r
    for i, a in enumerate(net.dec_rg):
        masks["dec%d" % (i + 1)] = pos(a, net.dec[i].site.order_out)
    if not net.affine:                                # GroupNorm blocks: three ReLUs each (lib/models.py:752-760)
        for i, b in enumerate(net.dec):
            for j, a in enumerate((b.A1, b.A2, b.A3)):
                masks["gn%d_%d" % (i + 1, j)] = pos(a, b.order_out)
    masks["dec_fc1"] = (net.dec_fc > 0).cpu()
    for i, a in enumerate(net.disc_act):
        r = sel(h["D_d"][i])
        for tag, sl in (("_real", slice(0, N)), ("_fake", slice(N, 2 * N))):
            masks["disc%d%s" % (i + 1, tag)] = pos(a[sl], net.disc[i].site.order_out)
            if r is not None:
                rows["disc%d%s" % (i + 1, tag)] = r
    masks["cond_pose_d"], masks["cond_pose_g"] = (net.cp_h[:N] > 0).cpu(), (net.cp_h[N:] > 0).cpu()
    masks["l1_sign"] = torch.sign(net.x_hat - net.in_x).cpu()     # sign decisions (-1, 0, +1) of the L1 reconstruction loss
    return masks, rows


def _oracle_update(h, cfg, params, mom, tb, step, dtype, ref_compat, masks=None, rows=None, record=None):
    """One O.train_update from numpy params/momentum (not modified); returns (result dict, new params, new momentum)."""
    from cape_b200 import topology as T
    o = O.Oracle(h["L"], h["D"], h["U"], h["L_d"], h["D_d"], cfg, dtype=dtype)
    if masks is not None:
        o.masks, o.mask_rows = masks, rows or {}
    o.record = record
    P = {k: torch.from_numpy(np.asarray(v)).to(dtype) for k, v in params.items()}
    M = {k: torch.from_numpy(np.asarray(v)).to(dtype) for k, v in mom.items()}
    ob = {k: v.to(dtype) for k, v in tb.items()}
    res = O.train_update(o, P, M, ob, step, T.smpl_edges(), ref_compat=ref_compat)
    return res, {k: v.numpy() for k, v in P.items()}, {k: v.numpy() for k, v in M.items()}


def train_step(h, cfg, N=2, ref_compat=False, step=100, seed=123, dtype=torch.float32, fc_scale=0.05,
               impose_masks=True, reorder=None, nsteps=1, use_graph=False, truth=False, report_unmasked=False):
    """Full VAE+GAN update(s) (BASELINE configs[2]): x_hat, losses, every gradient, the clipped momentum update and
    every post-update parameter vs the oracle's autograd, for `nsteps` CONSECUTIVE updates (the oracle carries its own
    parameters and momentum from update to update; fresh eps and batches every update as in CAPE.fit).

    impose_masks: the oracle's (leaky-)ReLUs take their branch decisions from the CUDA forward (about 1e-6 of all
    units sit within fp32 rounding of zero and would otherwise flip between any two fp32 implementations, which
    moves single-sample gradients such as the fc1 columns by percents); forward outputs and losses are compared
    unmasked in either case (keys "unmasked ...").
    use_graph: the CUDA step replays the two captured CUDA graphs (what bench.py times) instead of eager launches.
    truth: the comparison target is the FLOAT64 oracle, and every entry is returned as a pair
    (err(CUDA, fp64), err(fp32 oracle, fp64)) -- the second one measured with the fp32 oracle's own branch decisions
    imposed on a second fp64 run -- so that the caller can require the CUDA path to be as close to the truth as a
    plain fp32 CPU implementation is (reference initialisers, fc_scale=1.0: logvar reaches +-10, the KL term 1e4).
    report_unmasked: also return the gradient errors against an oracle WITHOUT imposed decisions ("unmasked grad ...",
    informational: they contain the sign flips)."""
    from cape_b200.network import CapeNetwork
    from cape_b200.params import param_specs
    from cape_b200.synthetic import make_batch
    p = [l.shape[0] for l in h["L"]]
    p_d = [l.shape[0] for l in h["L_d"]]
    specs = param_specs(cfg, p, p_d)
    params = calibrated_params(specs, seed, fc_scale)
    net = CapeNetwork(h["L"], h["D"], h["U"], h["L_d"], h["D_d"], cfg, N, params=params, ref_compat=ref_compat,
                      reorder=reorder)
    odt = torch.float64 if truth else dtype
    o_params = {k: np.asarray(v, np.float64 if truth else np.float32) for k, v in params.items()}
    o_mom = {k: np.zeros_like(v) for k, v in o_params.items()}
    out = {}
    for it in range(nsteps):
        batch = make_batch(N, cfg["nz"], seed=seed + 1000 * it)
        tb = {k: torch.from_numpy(v) for k, v in batch.items()}
        net.set_inputs(tb["x_g"], tb["cond_g"], tb["cond2_g"], tb["eps"], tb["x_d"], tb["cond_d"], tb["cond2_d"])
        if use_graph and it == 0:
            net.train_step(step=step, update=False)          # lazy initialisations before the capture
            torch.cuda.synchronize()
            net.capture_graphs()
        net.train_step(step=step + it, use_graph=use_graph)
        torch.cuda.synchronize()
        got_loss = net.loss_dict()
        got_x = net.x_hat.cpu().numpy()
        got_g = net.get_grads()
        got_p = net.get_params()
        got_m = net.PG.export(net.PG.mom)
        got_m.update(net.PD.export(net.PD.mom))
        masks, rows = cuda_masks(net, h, N) if impose_masks else (None, None)
        pre = "" if nsteps == 1 else "update %d: " % (it + 1)
        bound = None
        if truth:
            # how far a plain fp32 CPU implementation is from the truth on the same update (its own decisions imposed)
            rec = {}
            r32, _, _ = _oracle_update(h, cfg, {k: v.astype(np.float32) for k, v in o_params.items()},
                                       {k: v.astype(np.float32) for k, v in o_mom.items()}, tb, step + it,
                                       torch.float32, ref_compat, record=rec)
            r64b, _, _ = _oracle_update(h, cfg, o_params, o_mom, tb, step + it, torch.float64, ref_compat, masks=rec)
            bound = {"x_hat (max-rel)": rel(r32["x_hat"].numpy(), r64b["x_hat"].numpy())}
            for k in r64b["grads"]:
                bound["grad " + k] = rel(r32["grads"][k].numpy(), r64b["grads"][k].numpy())
        if report_unmasked and impose_masks:
            ru, _, _ = _oracle_update(h, cfg, o_params, o_mom, tb, step + it, odt, ref_compat)
            out[pre + "unmasked fwd x_hat (vertex-L2)"] = vertex_l2(got_x, ru["x_hat"].numpy())
            out[pre + "unmasked fwd x_hat (max-rel)"] = rel(got_x, ru["x_hat"].numpy())
            for k in ("recon", "edge", "latent", "gan_g", "gan_d"):
                out[pre + "unmasked fwd loss " + k] = abs(got_loss[k] - ru[k]) / max(abs(ru[k]), 1e-30)
            for k, g in ru["grads"].items():
                out[pre + "unmasked grad " + k] = rel(got_g[k].reshape(-1), g.numpy().reshape(-1))
        res, o_params, o_mom = _oracle_update(h, cfg, o_params, o_mom, tb, step + it, odt, ref_compat, masks, rows)
        cur = {"x_hat (vertex-L2)": vertex_l2(got_x, res["x_hat"].numpy()),
               "x_hat (max-rel)": rel(got_x, res["x_hat"].numpy())}
        for k in ("recon", "edge", "latent", "gan_g", "gan_d"):
            cur["loss " + k] = abs(got_loss[k] - res[k]) / max(abs(res[k]), 1e-30)
        for k, g in res["grads"].items():
            cur["grad " + k] = rel(got_g[k].reshape(-1), g.numpy().reshape(-1))
        for k, m in res["mom"].items():                  # momentum accumulator (first update: clip coefficient * grad)
            cur["clipped-update " + k] = rel(got_m[k].reshape(-1), m.numpy().reshape(-1))
        adam = "adam_v" in res
        if adam:                                         # Adam's second-moment slots
            got_v = net.PG.export(net.PG.var)
            got_v.update(net.PD.export(net.PD.var))
            for k, v in res["adam_v"].items():      # v is quadratic in g: half its relative error is the gradient's
                cur["adam-v " + k] = 0.5 * rel(got_v[k].reshape(-1), v.numpy().reshape(-1))
        for k, v in o_params.items():                    # post-update parameters (fp32 resolution of the weights)
            a, b = got_p[k].reshape(-1), v.reshape(-1)
            if adam:
                # Adam's step lr_t m / (sqrt(v) + eps) is +-lr for ANY gradient magnitude above eps, so an element whose
                # gradient lies within the parity tolerance of zero moves by a full step in a direction decided by
                # rounding: the parameters are compared where the gradient is resolved (|g| > 5 % of the tensor's max)
                g = np.abs(res["grads"][k].numpy().reshape(-1))
                keep = g > 0.05 * g.max()
                if not keep.any():
                    continue
                a, b = a[keep], b[keep]
            cur["param " + k] = rel(a, b)
        for k, v in cur.items():
            out[pre + k] = (v, bound.get(k, 0.0)) if truth else v
    return out


def set_tensor_cores(on):
    from cape_b200 import _lib
    return _lib.load().cape_set_tensor_cores(1 if on else 0)


def tc_vs_simt(h):
    """wgmma (3xTF32) kernels vs the fp32 SIMT kernels of the same entry points (forward, dX, dW), on layer
    shapes of the network and at row counts large enough to take the tensor-core weight-gradient path."""
    from cape_b200 import ops
    out = {}
    g = torch.Generator(device="cuda").manual_seed(5)
    cases = [("enc conv4 L3 128->128 K=2 +pool", h["L"][3], 2, 128, 128, 4, None, h["D"][3]),
             ("enc conv8 L7 512->512 K=2", h["L"][7], 2, 512, 512, 8, None, None),
             ("dec-like L5 320->128 K=2 +unpool", h["L"][5], 2, 320, 128, 3, h["U"][5], None),
             ("disc conv2 Ld1 64->64 K=3 +pool", h["L_d"][1], 3, 64, 64, 5, None, h["D_d"][1]),
             ("enc conv5 L4 128->256 K=2", h["L"][4], 2, 128, 256, 4, None, None),
             ("top L0 64->32 K=2", h["L"][0], 2, 64, 32, 2, None, None)]
    for tag, L, K, Fin, Fout, N, U, D in cases:
        Min = U.shape[1] if U is not None else L.shape[0]
        x = torch.randn(N, Min, Fin, device="cuda", generator=g)
        W = torch.randn(Fin * K, Fout, device="cuda", generator=g) * 0.1
        b = torch.randn(Fout, device="cuda", generator=g) * 0.1
        res = {}
        prev = set_tensor_cores(True)
        for on in (True, False):
            set_tensor_cores(on)
            xc, Wc = x.clone().requires_grad_(True), W.clone().requires_grad_(True)
            # no activation here: a (leaky-)ReLU would make dX/dW depend on sign flips of near-zero outputs between the
            # two contractions (see Oracle.masks), which is not what this comparison is about
            y = ops.chebyshev5(xc, L, Wc, K, bias=b, activation=None, pool=D, unpool=U)
            if on:
                dy = torch.randn(y.shape, device="cuda", generator=g)
            y.backward(dy)
            res[on] = (y.detach().cpu().numpy(), xc.grad.cpu().numpy(), Wc.grad.cpu().numpy())
        set_tensor_cores(prev)
        for nm, a, bb in zip(("fwd", "dx", "dW"), res[True], res[False]):
            out["tc-vs-simt %s %s" % (tag, nm)] = rel(a, bb)
    return out


def generator_forward(h, cfg, N=32, seed=123, fc_scale=1.0):
    """BASELINE configs[1]: condition nets + encoder + sampling + decoder forward at batch N vs the oracle (no imposed
    decisions: forward outputs only)."""
    from cape_b200.network import CapeNetwork
    from cape_b200.params import param_specs
    from cape_b200.synthetic import make_batch
    specs = param_specs(cfg, [l.shape[0] for l in h["L"]], [l.shape[0] for l in h["L_d"]])
    params = calibrated_params(specs, seed, fc_scale)
    net = CapeNetwork(h["L"], h["D"], h["U"], h["L_d"], h["D_d"], cfg, N, params=params)
    tb = {k: torch.from_numpy(v) for k, v in make_batch(N, cfg["nz"], seed=seed).items()}
    net.set_inputs(tb["x_g"], tb["cond_g"], tb["cond2_g"], tb["eps"])
    got = net.forward_generator().cpu().numpy()
    o = O.Oracle(h["L"], h["D"], h["U"], h["L_d"], h["D_d"], cfg)
    P = {k: torch.from_numpy(v) for k, v in params.items()}
    with torch.no_grad():
        y, y2 = o.cond_embeddings(tb["cond_g"], tb["cond2_g"], P)
        x_hat, zm, zl = o.generator(tb["x_g"], y, y2, tb["eps"], P)
    return {"x_hat (vertex-L2)": vertex_l2(got, x_hat.numpy()), "x_hat (max-rel)": rel(got, x_hat.numpy()),
            "z_mean": rel(net.z_mean.cpu().numpy(), zm.numpy()), "z_logvar": rel(net.z_logvar.cpu().numpy(), zl.numpy())}


def adam_kernel_case(n=100003, seed=5):
    """cape_adam_clip_update against the formula of tf.train.AdamOptimizer in float64 (two consecutive applications,
    with and without an active global-norm clip)."""
    import ctypes as C
    from cape_b200 import _lib
    lib = _lib.load()
    rng = np.random.RandomState(seed)
    out = {}
    for tag, gscale in (("clip inactive", 1e-3), ("clip active", 1.0)):
        w = rng.randn(n).astype(np.float32) * 0.1
        m, v = np.zeros(n, np.float64), np.zeros(n, np.float64)
        wd, md, vd = _cuda(w), torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
        w64 = w.astype(np.float64)
        # the hyper-parameters as the float32 values the kernel (and TF) see: 1 - fl32(0.999) differs from 1e-3 by 1.3e-5
        b1, b2, eps, lr, clip = float(np.float32(0.9)), float(np.float32(0.999)), 1e-8, 3e-3, 5.0
        for t in (1, 2):
            g = (rng.randn(n) * gscale).astype(np.float32)
            gd = _cuda(g)
            ss = torch.zeros(1, device="cuda")
            st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
            _lib.check(lib.cape_sumsq(C.c_void_p(gd.data_ptr()), n, C.c_void_p(ss.data_ptr()), st))
            lr_t = lr * np.sqrt(1 - b2 ** t) / (1 - b1 ** t)
            lrd = torch.tensor([lr_t], dtype=torch.float32, device="cuda")
            _lib.check(lib.cape_adam_clip_update(C.c_void_p(wd.data_ptr()), C.c_void_p(gd.data_ptr()),
                                                 C.c_void_p(md.data_ptr()), C.c_void_p(vd.data_ptr()), n,
                                                 C.c_void_p(ss.data_ptr()), clip, C.c_void_p(lrd.data_ptr()), b1, b2, eps, st))
            g64 = g.astype(np.float64)
            coef = clip / max(np.sqrt((g64 ** 2).sum()), clip)
            gc = coef * g64
            m = b1 * m + (1 - b1) * gc
            v = b2 * v + (1 - b2) * gc * gc
            w64 = w64 - lr_t * m / (np.sqrt(v) + eps)
        torch.cuda.synchronize()
        out["adam %s: m" % tag] = rel(md.cpu().numpy(), m)
        out["adam %s: v" % tag] = rel(vd.cpu().numpy(), v)
        out["adam %s: w" % tag] = rel(wd.cpu().numpy(), w64)
    return out


def compare_with_reference_golden(tag, x_hat, losses, params_after):
    """Relative errors of an update's results against tests/golden/ref_models_golden.npz -- the numbers the REFERENCE's
    own lib/models.py produced on the TF shim (tests/golden/make_ref_golden.py) for the inputs of `reference_golden_inputs`.
    Pure numpy (tests/test_reference_golden.py runs it on the oracle's results on CPU, the GPU test on the CUDA path's)."""
    import make_ref_golden as G
    z = G.load()
    out = {"x_hat (vertex-L2)": vertex_l2(x_hat, z[tag + "/x_hat"]), "x_hat (max-rel)": rel(x_hat, z[tag + "/x_hat"])}
    for k in ("recon", "edge", "latent", "gan_g", "gan_d"):
        want = float(z["%s/%s" % (tag, k)])
        out["loss " + k] = abs(losses[k] - want) / max(abs(want), 1e-30)
    for name, v in params_after.items():
        base = "%s/params_after/%s" % (tag, name)
        v = np.asarray(v, np.float32).reshape(-1)
        if base + "#full" in z.files:
            out["param " + name] = rel(v, z[base + "#full"].reshape(-1))
        else:
            out["param " + name] = rel(v[G.sample_index(name, v.size)], z[base + "#sample"])
    return out


def reference_golden_update(h, tag="nz64"):
    """The update the reference golden file holds (affine nz64 model, batch 2, global_step 100, the reference's own
    optimiser wiring = ref_compat) on the CUDA path, compared with the reference's numbers directly."""
    import make_ref_golden as G
    from cape_b200.network import CapeNetwork
    cfg, N, step = next((c, n, s) for t, c, n, s in G.configs() if t == tag)
    params, batch = G.inputs(cfg, h, N)
    net = CapeNetwork(h["L"], h["D"], h["U"], h["L_d"], h["D_d"], cfg, N, params=params, ref_compat=True)
    tb = {k: torch.from_numpy(v) for k, v in batch.items()}
    net.set_inputs(tb["x_g"], tb["cond_g"], tb["cond2_g"], tb["eps"], tb["x_d"], tb["cond_d"], tb["cond2_d"])
    net.train_step(step=step)
    torch.cuda.synchronize()
    # Forward-side quantities and the discriminator's parameters only.  The reference took its OWN (leaky-)ReLU branch
    # decisions, and the few pre-activations within fp32 rounding of zero fall on the other side in any other fp32
    # implementation (see train_step: that is why gradients are compared with imposed decisions); gradients jump there,
    # and a zero-initialised bias after one update IS its gradient (times -lr), so the generator's post-update
    # parameters are not compared here -- the first run of this test with them failed for that reason.  The
    # discriminator's update under the reference's wiring (lib/models.py:466) involves no gradient at all.
    after = {k: v for k, v in net.get_params().items() if k.startswith("discriminator")}
    return compare_with_reference_golden(tag, net.x_hat.cpu().numpy(), net.loss_dict(), after)
