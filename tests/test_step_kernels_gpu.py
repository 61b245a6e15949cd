"""The small kernels of every training step, called through the C ABI at their edge shapes and compared with a float64
NumPy / torch computation of the same operation:

- group norm + ReLU (groupnorm.cu, cape_gn_relu_fwd / _bwd): every (C, rows) pair of the GroupNorm decoder blocks,
  groups of 1 to 17 channels, the batch-64 grid-stride wrap, the API edges of the row-slot layout, data far from zero
  and condition channels that are constant over the vertices, accumulation into prefilled gradients, rejections;
- the losses, sampling, optimiser and copy kernels of misc.cu;
- cape_gemm off its usual paths: the scalar kernel on the vectorised kernel's layouts, split-K limited or switched off
  by the workspace, beta != 0 with split-K, ReLU, C inside a wider row.

Every output buffer is followed by sentinels that must be unchanged, and every call's number of launches is checked
with cape_launch_count."""
import contextlib
import ctypes as C

import numpy as np
import pytest
import scipy.sparse as sp
import torch

pytestmark = pytest.mark.gpu

GUARD = 67            # sentinel floats after every output buffer
NAN = np.float32("nan")
EPS = 1e-5


def _E():
    from cape_b200 import engine
    return engine


def _lib():
    from cape_b200 import _lib
    return _lib.load()


def _dev():
    return torch.device("cuda", 0)


def _tp():
    from cape_b200 import ops
    return ops.topology_for(_dev())


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


@contextlib.contextmanager
def _knobs(tuning=()):
    """Sets process-wide kernel-selection knobs for the duration of a block and always restores them."""
    lib, undo = _lib(), []
    try:
        for k, v in tuning:
            prev = lib.cape_set_tuning(k, v)
            undo.append(lambda k=k, prev=prev: lib.cape_set_tuning(k, prev))
        yield
    finally:
        for u in reversed(undo):
            u()


def _launches(fn):
    """Runs fn() to completion; returns (its return value, the number of kernels the library launched)."""
    lib = _lib()
    torch.cuda.synchronize()
    n0 = lib.cape_launch_count()
    rc = fn()
    torch.cuda.synchronize()
    return rc, lib.cape_launch_count() - n0


def _buf(init, head=0, fill=NAN):
    """A flat device buffer: `head` sentinels, the values of `init`, GUARD sentinels.  Returns (buffer, view of the
    target with init's shape, host copy of the whole buffer)."""
    init = np.asarray(init, np.float32)
    host = np.full(head + init.size + GUARD, fill, np.float32)
    host[head:head + init.size] = init.ravel()
    d = torch.from_numpy(host).to(_dev())
    return d, d[head:head + init.size].view(init.shape), host


def _guard_ok(d, host, head=0, n=None, what=""):
    got = d.cpu().numpy()
    n = host.size - head - GUARD if n is None else n
    out = np.concatenate([got[:head], got[head + n:]])
    ref = np.concatenate([host[:head], host[head + n:]])
    assert np.array_equal(out, ref, equal_nan=True), "%s: wrote outside its target" % what


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def _report(case, err):
    print("worst-rel-err %-64s %.3e" % (case, err))


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(_dev())


# ---------------------------------------------------------------------------------------------------------------------
# group norm + ReLU
# ---------------------------------------------------------------------------------------------------------------------
def _gn_truth(x, gm, bt, dy, G, mask, dtype):
    """Oracle.gn + ReLU in `dtype` with torch autograd; the ReLU decisions of the backward pass are `mask` (the CUDA
    y > 0), so the comparison is not about sign flips of near-zero outputs."""
    from oracle import cape_oracle as O
    o = O.Oracle([], [], [], [], [], dict(F=[x.shape[2]], K=[2], Kd=3))
    xt, gt, btt = (torch.from_numpy(a).to(dtype).requires_grad_(True) for a in (x, gm, bt))
    z = o.gn(xt, gt, btt, G=G, eps=EPS)
    (z * torch.from_numpy(mask).to(dtype) * torch.from_numpy(dy).to(dtype)).sum().backward()
    return {"y": torch.relu(z).detach().double().numpy(), "dx": xt.grad.double().numpy(),
            "dgamma": gt.grad.double().numpy(), "dbeta": btt.grad.double().numpy()}


def _gn_stats64(x, G):
    N, rows, Cc = x.shape
    xg = x.astype(np.float64).reshape(N, rows, G, Cc // G)
    mean = xg.mean(axis=(1, 3))
    var = ((xg - mean[:, None, :, None]) ** 2).mean(axis=(1, 3))
    return mean, var


def gn_call(x, gm, bt, dy, G, tp=None, dx0=None, dg0=None, db0=None):
    """Forward and backward through the C ABI; returns the outputs (numpy) after checking launches and sentinels."""
    tp = tp or _tp()
    lib = tp.lib
    N, rows, Cc = x.shape
    xd, gd, bd, dyd = _cuda(x), _cuda(gm), _cuda(bt), _cuda(dy)
    yb, y, yh = _buf(np.full(x.shape, NAN))
    sb, stats, sh = _buf(np.full((N, G, 2), NAN))
    accumulate = dx0 is not None
    xb, dx, xh = _buf(dx0 if accumulate else np.full(x.shape, NAN))
    gb, dg, gh = _buf(np.zeros(Cc) if dg0 is None else dg0)
    bb, db, bh = _buf(np.zeros(Cc) if db0 is None else db0)
    rc, n = _launches(lambda: lib.cape_gn_relu_fwd(tp.h, _p(xd), N, rows, Cc, G, EPS, _p(gd), _p(bd), _p(y), _p(stats),
                                                   _st()))
    assert rc == 0 and n == 3, (rc, n)
    rc, n = _launches(lambda: lib.cape_gn_relu_bwd(tp.h, _p(xd), _p(y), _p(dyd), N, rows, Cc, G, _p(gd), _p(stats),
                                                   _p(dx), 1 if accumulate else 0, _p(dg), _p(db), _st()))
    assert rc == 0 and n == 2, (rc, n)
    for d, h, what in ((yb, yh, "y"), (sb, sh, "stats"), (xb, xh, "dx"), (gb, gh, "dgamma"), (bb, bh, "dbeta")):
        _guard_ok(d, h, what="gn " + what)
    return {"y": y.cpu().numpy(), "stats": stats.cpu().numpy(), "dx": dx.cpu().numpy(), "dgamma": dg.cpu().numpy(),
            "dbeta": db.cpu().numpy()}


def gn_case(case, x, G, *, gm=None, bt=None, seed=0, prefill=False, tp=None):
    """Checks y, dx, dgamma, dbeta against float64 (error at most max(1e-4, twice that of the float32 Oracle.gn)) and
    the statistics against a float64 two-pass (rstd relative error <= 1e-5, mean error <= 1e-6 max(|mean|, std))."""
    rng = np.random.RandomState(seed + 1000)
    N, rows, Cc = x.shape
    gm = rng.normal(1, 0.2, size=Cc).astype(np.float32) if gm is None else gm
    bt = rng.normal(0, 0.2, size=Cc).astype(np.float32) if bt is None else bt
    dy = rng.normal(size=x.shape).astype(np.float32)
    pre = {}
    if prefill:
        pre["dx"] = rng.normal(size=x.shape).astype(np.float32)
        pre["dgamma"] = rng.normal(size=Cc).astype(np.float32)
        pre["dbeta"] = rng.normal(size=Cc).astype(np.float32)
    out = gn_call(x, gm, bt, dy, G, tp=tp, dx0=pre.get("dx"), dg0=pre.get("dgamma"), db0=pre.get("dbeta"))
    mask = out["y"] > 0
    t64 = _gn_truth(x, gm, bt, dy, G, mask, torch.float64)
    t32 = _gn_truth(x, gm, bt, dy, G, mask, torch.float32)
    if prefill:
        for k, v in pre.items():
            t64[k] = t64[k] + v.astype(np.float64)
            t32[k] = (t32[k].astype(np.float32) + v).astype(np.float64)
    errs = {}
    for k in ("y", "dx", "dgamma", "dbeta"):
        assert np.isfinite(out[k]).all(), "%s: %s not finite" % (case, k)
        errs[k] = (_rel(out[k], t64[k]), _rel(t32[k], t64[k]))
    mean, var = _gn_stats64(x, G)
    rstd = 1.0 / np.sqrt(var + EPS)
    e_rstd = np.abs(out["stats"][..., 1] / rstd - 1.0)
    e_mean = np.abs(out["stats"][..., 0] - mean) / np.maximum(np.abs(mean), np.sqrt(var))
    print("gn %-44s rstd %.2e (group %s)  mean %.2e  y %.2e/%.2e dx %.2e/%.2e dgamma %.2e/%.2e dbeta %.2e/%.2e" % (
        case, e_rstd.max(), np.unravel_index(e_rstd.argmax(), e_rstd.shape), e_mean.max(),
        *errs["y"], *errs["dx"], *errs["dgamma"], *errs["dbeta"]))
    assert e_rstd.max() <= 1e-5, "%s: rstd relative error %.3e" % (case, e_rstd.max())
    assert e_mean.max() <= 1e-6, "%s: mean error %.3e x max(|mean|, std)" % (case, e_mean.max())
    for k, (e, e32) in errs.items():
        assert e <= max(1e-4, 2 * e32), "%s: %s error %.3e (float32 Oracle.gn: %.3e)" % (case, k, e, e32)


def _gn_x(N, rows, Cc, seed, mu=0.3, sigma=1.5):
    rng = np.random.RandomState(seed)
    return (mu + sigma * rng.normal(size=(N, rows, Cc))).astype(np.float32)


@pytest.fixture(scope="module")
def gn_blocks(hierarchy):
    """(C, G, rows, U, condition channels) of every group norm of the decoder blocks of the nz18 network (GroupNorm
    decoder), in order; the first group norm of a block normalises its input and condition channels."""
    from cape_b200.network import CapeNetwork
    from cape_b200.params import NZ18_PLAIN
    h = hierarchy
    net = CapeNetwork(h["L"], h["D"], h["U"], h["L_d"], h["D_d"], dict(NZ18_PLAIN, decay_steps=10), batch_size=1)
    out = []
    for i, blk in enumerate(net.dec):
        U = h["U"][-i - 1]
        assert U.shape[0] == blk.rows
        out += [(g["C"], g["G"], blk.rows, U, blk.Cc if j == 0 else 0) for j, g in enumerate(blk.gn)]
    del net
    torch.cuda.synchronize()
    return out


def test_gn_model_shapes(gn_blocks):
    """Every (C, rows) pair the GroupNorm decoder runs, at N = 2: channels per group 17, 9, 8, 5, 4, 3, 2, 1."""
    pairs = sorted({(Cc, G, rows) for Cc, G, rows, _, _ in gn_blocks})
    assert len(pairs) >= 8 and {Cc // G for Cc, G, _ in pairs} >= {17, 9, 8, 5, 4, 3, 2, 1}, pairs
    for i, (Cc, G, rows) in enumerate(pairs):
        gn_case("C=%d G=%d rows=%d N=2" % (Cc, G, rows), _gn_x(2, rows, Cc, i), G, seed=i)


@pytest.mark.parametrize("Cc,rows", [(160, 1723), (96, 6890)])
def test_gn_batch64(Cc, rows):
    """The benchmark batch: the apply kernels' grid cap makes their grid-stride loops wrap."""
    bx = (rows * Cc // 4 + 255) // 256
    assert bx > (_sms() * 16 + 63) // 64
    gn_case("C=%d rows=%d N=64" % (Cc, rows), _gn_x(64, rows, Cc, Cc), 32, seed=Cc)


# C = 4 / 8 / 12 with one channel per group (the 32-slot cap on row slots), C = 36 / G = 12 (28 row slots: does not
# divide 256), C = 1024 (one row slot, all 256 threads); rows of 1 and around the 64-row block
@pytest.mark.parametrize("Cc,G,rows", [(4, 4, 300), (8, 8, 300), (12, 12, 300), (36, 12, 300), (1024, 32, 100),
                                       (96, 32, 1), (96, 32, 63), (96, 32, 64), (96, 32, 65),
                                       (36, 12, 1), (36, 12, 63), (36, 12, 64), (36, 12, 65)])
def test_gn_api_edges(Cc, G, rows):
    gn_case("C=%d G=%d rows=%d N=3" % (Cc, G, rows), _gn_x(3, rows, Cc, Cc + rows), G, seed=rows)


# data far from zero: x = mu + sigma N(0, 1)
@pytest.mark.parametrize("ratio", [10, 100, 1000])
@pytest.mark.parametrize("Cc,rows", [(544, 862), (256, 431), (96, 6890)])
def test_gn_offset(Cc, rows, ratio):
    sigma = 0.7
    gn_case("offset C=%d rows=%d mean/std=%d" % (Cc, rows, ratio), _gn_x(2, rows, Cc, ratio + Cc, ratio * sigma, sigma),
            32, seed=ratio)


# the first group norm of a decoder block normalises [x ; rowsum(U) c]: the condition channels are constant over the
# vertices up to rowsum(U), and the last groups hold nothing else (the widest level of each width)
@pytest.mark.parametrize("Cc", [544, 160, 96])
def test_gn_condition_groups(gn_blocks, Cc):
    _, G, rows, U, Cond = [b for b in gn_blocks if b[0] == Cc and b[4]][-1]
    assert Cond == 32
    rng = np.random.RandomState(Cc)
    N = 2
    x = rng.normal(size=(N, rows, Cc)).astype(np.float32)
    c = (1 + 0.01 * rng.normal(size=(N, Cond))).astype(np.float32)
    rs = np.asarray(sp.csr_matrix(U).astype(np.float32).sum(axis=1), np.float32).ravel()
    x[:, :, Cc - Cond:] = rs[None, :, None] * c[:, None, :]
    gn_case("condition C=%d rows=%d" % (Cc, rows), x, G, seed=Cc)


def test_gn_gamma_sign():
    """Negative and zero gamma (the ReLU mask then selects other elements than the normalised sign)."""
    rng = np.random.RandomState(3)
    for Cc, rows in ((544, 216), (96, 862)):
        gm = rng.normal(size=Cc).astype(np.float32)
        gm[::5] = 0.0
        gm[1::5] = -np.abs(gm[1::5])
        gn_case("gamma +/-/0 C=%d rows=%d" % (Cc, rows), _gn_x(2, rows, Cc, 7), 32, gm=gm, seed=Cc)


@pytest.mark.parametrize("Cc,G,rows", [(544, 32, 216), (96, 32, 6890), (36, 12, 65)])
def test_gn_accumulate(Cc, G, rows):
    """accumulate_dx = 1 into a prefilled dx; dgamma / dbeta add into prefilled values."""
    gn_case("accumulate C=%d rows=%d" % (Cc, rows), _gn_x(2, rows, Cc, 11), G, seed=5, prefill=True)


def test_gn_rejections():
    """Shapes the kernels cannot run return rc < 0, launch nothing and write nothing; a handle whose workspace is one
    byte short of N G 16 bytes is refused and one with exactly that much runs."""
    E = _E()
    rng = np.random.RandomState(0)

    def attempt(tp, N, rows, Cc, G):
        x = _gn_x(N, rows, Cc, 1)
        xd, dyd = _cuda(x), _cuda(rng.normal(size=x.shape).astype(np.float32))
        gd, bd = _cuda(np.ones(Cc, np.float32)), _cuda(np.zeros(Cc, np.float32))
        yb, y, yh = _buf(np.full(x.shape, NAN))
        sb, st, sh = _buf(np.full((N, max(G, 1), 2), NAN))
        xb, dx, xh = _buf(np.full(x.shape, NAN))
        gb, dg, gh = _buf(np.full(Cc, 7.0))
        bb, db, bh = _buf(np.full(Cc, 7.0))
        rf, nf = _launches(lambda: tp.lib.cape_gn_relu_fwd(tp.h, _p(xd), N, rows, Cc, G, EPS, _p(gd), _p(bd), _p(y),
                                                           _p(st), _st()))
        rb, nb = _launches(lambda: tp.lib.cape_gn_relu_bwd(tp.h, _p(xd), _p(xd), _p(dyd), N, rows, Cc, G, _p(gd),
                                                           _p(st), _p(dx), 0, _p(dg), _p(db), _st()))
        return (rf, nf, rb, nb), [(yb, yh), (sb, sh), (xb, xh), (gb, gh), (bb, bh)]

    for (N, rows, Cc, G) in ((2, 100, 6, 2), (2, 100, 40, 32), (2, 100, 132, 33)):
        (rf, nf, rb, nb), bufs = attempt(_tp(), N, rows, Cc, G)
        assert rf < 0 and rb < 0 and nf == 0 and nb == 0, (Cc, G, rf, rb, nf, nb)
        for d, h in bufs:
            _guard_ok(d, h, n=0, what="rejected gn C=%d G=%d" % (Cc, G))
    N, G = 3, 32
    tp = E.Topology(0)
    tp.reserve_workspace(N * G * 16 - 1)
    (rf, nf, rb, nb), bufs = attempt(tp, N, 100, 96, G)
    assert rf < 0 and rb < 0 and nf == 0 and nb == 0, (rf, rb, nf, nb)
    for d, h in bufs:
        _guard_ok(d, h, n=0, what="gn with a short workspace")
    tp2 = E.Topology(0)
    tp2.reserve_workspace(N * G * 16)
    gn_case("workspace of exactly N G 16 bytes", _gn_x(N, 100, 96, 2), G, tp=tp2)


# ---------------------------------------------------------------------------------------------------------------------
# misc.cu: losses
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def nbr(hierarchy):
    """The level-0 neighbour operator of the reconstruction loss (as the network registers it)."""
    from cape_b200.network import _adjacency
    A = sp.csr_matrix(_adjacency(hierarchy["L"][0]))
    return A, _tp().add_operator(A), int(A.nnz // 2)


def _recon_truth(pred, gt, A, n_edges, lam_l1, lam_edge):
    N, rows, _ = pred.shape
    res = pred.astype(np.float64) - gt.astype(np.float64)
    cnt, ecnt = N * rows * 3.0, float(N * n_edges)
    r_idx = np.repeat(np.arange(rows), np.diff(A.indptr))
    e = res[:, r_idx] - res[:, A.indices]                           # [N, nnz, 3]: every edge from both ends
    ln = np.sqrt((e ** 2).sum(-1))
    w = np.where(ln[..., None] > 0, e / np.where(ln > 0, ln, 1.0)[..., None], 0.0)
    S = sp.csr_matrix((np.ones(r_idx.size), (r_idx, np.arange(r_idx.size))), shape=(rows, r_idx.size))
    ge = (S @ w.transpose(1, 0, 2).reshape(r_idx.size, N * 3)).reshape(rows, N, 3).transpose(1, 0, 2)
    grad = lam_l1 / cnt * np.sign(res) + lam_edge / ecnt * ge
    return np.abs(res).sum() / cnt, ln.sum() * 0.5 / ecnt, grad


@pytest.mark.parametrize("N", [2, 64])
@pytest.mark.parametrize("lam_edge", [0.0, 0.7])
@pytest.mark.parametrize("kl", [True, False])
def test_recon_losses(nbr, N, lam_edge, kl):
    """L1 + edge-length losses and their gradient (accumulated into prefilled values), and the KL term (into a
    non-zero start, its grid-stride loop wrapping at N nz > 64 x 256; mean / logvar NULL: the KL slot is untouched).
    Some residual components are exactly 0 (zero L1 gradient), some vertices have the residual of a neighbour
    (zero-length edges: nothing may be NaN)."""
    tp = _tp()
    A, op, n_edges = nbr
    rows = A.shape[0]
    assert (N * rows) % 256
    rng = np.random.RandomState(N)
    gt = rng.normal(size=(N, rows, 3)).astype(np.float32)
    pred = (gt + 0.1 * rng.normal(size=gt.shape)).astype(np.float32)
    zero = rng.choice(rows, 40, replace=False)
    pred[:, zero, 1] = gt[:, zero, 1]
    pred[0, zero[:10], :] = gt[0, zero[:10], :]
    twins = list(zero)
    for v in rng.choice(rows, 30, replace=False):
        u = A.indices[A.indptr[v]]
        if v not in twins and u not in twins:
            pred[:, v], gt[:, v] = pred[:, u], gt[:, u]
            twins += [v, u]
    l1, le, grad = _recon_truth(pred, gt, A, n_edges, 1.0, lam_edge)
    gscale = np.abs(grad).max()
    d0 = (gscale * rng.normal(size=grad.shape)).astype(np.float32)
    l0 = np.array([0.5 * l1, 0.3, 1.7], np.float32)
    nz = 300 if N == 64 else 18
    mean = rng.normal(size=(N, nz)).astype(np.float32)
    logvar = rng.uniform(-10, 10, size=(N, nz)).astype(np.float32)
    m64, lv64 = mean.astype(np.float64), logvar.astype(np.float64)
    klv = (-0.5 * (1 + lv64 - m64 ** 2 - np.exp(lv64))).sum() / N
    pd, gd = _cuda(pred), _cuda(gt)
    db, dpred, dh = _buf(d0)
    lb, losses, lh = _buf(l0)
    md, lvd = (_cuda(mean), _cuda(logvar)) if kl else (None, None)
    rc, n = _launches(lambda: tp.lib.cape_recon_losses(tp.h, op, _p(pd), _p(gd), N, rows, 1.0, lam_edge, n_edges,
                                                        _p(md), _p(lvd), nz if kl else 0, _p(dpred), _p(losses),
                                                        _st()))
    assert rc == 0 and n == (2 if kl else 1), (rc, n)
    _guard_ok(db, dh, what="dpred")
    _guard_ok(lb, lh, what="losses")
    got, lg = dpred.cpu().numpy(), losses.cpu().numpy().astype(np.float64)
    assert np.isfinite(got).all() and np.isfinite(lg).all()
    want = d0.astype(np.float64) + grad
    err = _rel(got, want)
    if lam_edge == 0:          # the zero residual components get no L1 gradient: dpred keeps its value exactly
        assert np.array_equal(got[:, zero, 1], d0[:, zero, 1])
    e_l1 = abs(lg[0] - (l0[0] + l1)) / (l0[0] + l1)
    e_le = abs(lg[1] - (l0[1] + le)) / (l0[1] + le)
    e_kl = abs(lg[2] - (l0[2] + klv)) / abs(l0[2] + klv) if kl else 0.0
    if not kl:
        assert lg[2] == l0[2], "the KL slot changed without mean / logvar"
    _report("recon N=%d lambda_edge=%g kl=%d: dpred / l1 / edge / kl %.1e %.1e %.1e %.1e" % (
        N, lam_edge, kl, err, e_l1, e_le, e_kl), max(err, e_l1, e_le, e_kl))
    assert err <= 1e-5 and e_l1 <= 1e-5 and e_le <= 1e-5 and e_kl <= 1e-5, (err, e_l1, e_le, e_kl)


def test_bce_logits():
    """Logits of +-100, +-20, 0 and random values, labels 0 / 0.1 / 0.9 / 1, n past the 256-block cap; dlogits or loss
    NULL."""
    lib = _lib()
    rng = np.random.RandomState(0)
    n = 256 * 256 + 4321
    x = rng.normal(0, 4, size=n).astype(np.float32)
    x[:10] = [100, -100, 20, -20, 0, 100, -100, 20, -20, 0]
    x[-5:] = [100, -100, 20, -20, 0]
    x64 = x.astype(np.float64)
    xd = _cuda(x)
    for label in (0.0, 0.1, 0.9, 1.0):
        lab = float(np.float32(label))
        scale = 0.37
        loss = (np.maximum(x64, 0) - x64 * lab + np.log1p(np.exp(-np.abs(x64)))).sum() / n
        grad = (1 / (1 + np.exp(-x64)) - lab) * scale / n
        for mode in ("both", "no-grad", "no-loss"):
            gb, g, gh = _buf(np.full(n, NAN))
            lb, ls, lh = _buf(np.array([2.5], np.float32))
            rc, k = _launches(lambda: lib.cape_bce_logits(_p(xd), n, label, scale, None if mode == "no-grad" else _p(g),
                                                          None if mode == "no-loss" else _p(ls), _st()))
            assert rc == 0 and k == 1
            _guard_ok(gb, gh, n=0 if mode == "no-grad" else n, what="dlogits")
            _guard_ok(lb, lh, n=0 if mode == "no-loss" else 1, what="loss")
            if mode != "no-grad":
                e = _rel(g.cpu().numpy(), grad)
                assert e <= 1e-5, (label, mode, e)
            if mode != "no-loss":
                e = abs(float(ls.cpu()) - (2.5 + loss)) / (2.5 + loss)
                assert e <= 1e-5, (label, mode, e)
        _report("bce label=%g" % label, e)


# ---------------------------------------------------------------------------------------------------------------------
# misc.cu: re-parameterisation
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N,nz,stride", [(7, 18, 50), (64, 18, 50), (3, 64, 128), (5, 13, 13)])
def test_vae_sample(N, nz, stride):
    """z = mean + exp(logvar / 2) eps into a row of the concat buffer (z_stride > nz), and its backward from a strided
    dz; logvar in +-10, N nz not a multiple of 256."""
    lib = _lib()
    rng = np.random.RandomState(nz + N)
    mean = rng.normal(size=(N, nz)).astype(np.float32)
    logvar = rng.uniform(-10, 10, size=(N, nz)).astype(np.float32)
    eps = rng.normal(size=(N, nz)).astype(np.float32)
    m64, lv64, e64 = (a.astype(np.float64) for a in (mean, logvar, eps))
    md, lvd, ed = _cuda(mean), _cuda(logvar), _cuda(eps)
    zb, z, zh = _buf(np.full((N, stride), NAN))
    rc, k = _launches(lambda: lib.cape_vae_sample_fwd(_p(md), _p(lvd), _p(ed), _p(z), stride, N, nz, _st()))
    assert rc == 0 and k == 1
    zg = zb.cpu().numpy()[:N * stride].reshape(N, stride)
    assert np.isnan(zg[:, nz:]).all(), "z: wrote past nz"
    _guard_ok(zb, zh, what="z")
    ez = _rel(zg[:, :nz], m64 + np.exp(lv64 / 2) * e64)
    dz = np.full((N, stride), NAN, np.float32)
    dz[:, :nz] = rng.normal(size=(N, nz))
    dzd = _cuda(dz)
    kl = 8e-4
    mb, dm, mh = _buf(np.full((N, nz), NAN))
    lb, dlv, lh = _buf(np.full((N, nz), NAN))
    rc, k = _launches(lambda: lib.cape_vae_sample_bwd(_p(dzd), stride, _p(md), _p(lvd), _p(ed), _p(dm), _p(dlv), N, nz,
                                                      kl, _st()))
    assert rc == 0 and k == 1
    _guard_ok(mb, mh, what="dmean")
    _guard_ok(lb, lh, what="dlogvar")
    d64 = dz[:, :nz].astype(np.float64)
    em = _rel(dm.cpu().numpy(), d64 + kl * m64 / N)
    el = _rel(dlv.cpu().numpy(), d64 * e64 * 0.5 * np.exp(lv64 / 2) + kl * 0.5 * (np.exp(lv64) - 1) / N)
    _report("vae N=%d nz=%d stride=%d" % (N, nz, stride), max(ez, em, el))
    assert max(ez, em, el) <= 1e-5, (ez, em, el)


# ---------------------------------------------------------------------------------------------------------------------
# misc.cu: global norm and the momentum update
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 3, 4, 5, 257, (1 << 20) + 3])
def test_sumsq(n):
    """The float4 body and the scalar tail; accumulation into a non-zero value; two calls in a row (the last block
    resets the completion counter) give the same bits."""
    lib = _lib()
    rng = np.random.RandomState(n % 1000)
    g = rng.normal(size=n).astype(np.float32)
    gd = _cuda(g)
    want = float((g.astype(np.float64) ** 2).sum())
    outs = []
    for start in (0.0, 3.25, 0.0):
        sb, s, sh = _buf(np.array([start], np.float32))
        rc, k = _launches(lambda: lib.cape_sumsq(_p(gd), n, _p(s), _st()))
        assert rc == 0 and k == 1
        _guard_ok(sb, sh, what="sumsq")
        got = float(s.cpu())
        e = abs(got - (start + want)) / (start + want)
        assert e <= 1e-5, (n, start, got, start + want)
        outs.append(got)
    assert outs[0] == outs[2], "two identical reductions differ: %r" % outs
    _report("sumsq n=%d" % n, e)


@pytest.mark.parametrize("n", [1, 3, 257, (1 << 20) + 3])
@pytest.mark.parametrize("clip", ["active", "inactive", "none"])
@pytest.mark.parametrize("momentum", [0.0, 0.9])
def test_sgd_clip_update(n, clip, momentum):
    """Two consecutive momentum updates with the global-norm clip active, inactive or off (sumsq NULL); the learning
    rate is read from device memory and changes between the steps."""
    lib = _lib()
    rng = np.random.RandomState(n % 997)
    w = rng.normal(size=n).astype(np.float32)
    mom = rng.normal(size=n).astype(np.float32)
    wb, wd, wh = _buf(w)
    mb, md, mh = _buf(mom)
    w64, m64 = w.astype(np.float64), mom.astype(np.float64)
    mom_f = float(np.float32(momentum))
    lr = torch.zeros(1, device=_dev())
    for step, lr_v in enumerate((0.05, 0.2)):
        g = rng.normal(size=n).astype(np.float32)
        gd = _cuda(g)
        g64 = g.astype(np.float64)
        norm = np.sqrt((g64 ** 2).sum())
        cn = {"active": 0.5 * norm, "inactive": 2.0 * norm + 1, "none": 1.0}[clip]
        ss = torch.zeros(1, device=_dev())
        assert lib.cape_sumsq(_p(gd), n, _p(ss), _st()) == 0
        lr.fill_(lr_v)
        coef = cn / max(norm, cn) if clip != "none" else 1.0
        rc, k = _launches(lambda: lib.cape_sgd_clip_update(_p(wd), _p(gd), _p(md), n, None if clip == "none" else _p(ss),
                                                           cn, _p(lr), momentum, _st()))
        assert rc == 0 and k == 1
        a = mom_f * m64 + coef * g64
        lr64 = float(np.float32(lr_v))
        w64, m64 = w64 - lr64 * a, a
        _guard_ok(wb, wh, what="w")
        _guard_ok(mb, mh, what="mom")
        mg, wg = md.cpu().numpy().astype(np.float64), wd.cpu().numpy().astype(np.float64)
        em = _rel(mg, m64)
        # w: the update against 1e-5 of the largest update, plus the rounding of w itself
        ew = float((np.abs(wg - w64) / (1e-5 * np.abs(lr64 * a).max() + 6e-8 * np.abs(w64))).max())
        assert em <= 1e-5 and ew <= 1.0, (step, em, ew)
        # the next step continues from the kernel's own state
        w64, m64 = wg, mg
    _report("sgd n=%d clip=%s momentum=%g" % (n, clip, momentum), em)


# ---------------------------------------------------------------------------------------------------------------------
# misc.cu: elementwise kernels and copies
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("alpha", [0.0, 0.2])
def test_act_bwd_axpy(alpha):
    """Grid-stride loops that wrap (n > 8 SMs 256, not a multiple of 256); y of exactly +0 and -0 takes the alpha
    branch.  act_bwd is one IEEE product, so it must match the float32 product exactly."""
    lib = _lib()
    rng = np.random.RandomState(int(alpha * 10))
    for n in (1001, 8 * _sms() * 256 + 777):
        y = rng.normal(size=n).astype(np.float32)
        y[::7] = 0.0
        y[3::7] = -0.0
        dy = rng.normal(size=n).astype(np.float32)
        yd, dyd = _cuda(y), _cuda(dy)
        gb, g, gh = _buf(np.full(n, NAN))
        rc, k = _launches(lambda: lib.cape_act_bwd(_p(dyd), _p(yd), _p(g), n, alpha, _st()))
        assert rc == 0 and k == 1
        _guard_ok(gb, gh, what="act_bwd")
        want = np.where(y > 0, dy, dy * np.float32(alpha))
        got = g.cpu().numpy()
        assert np.array_equal(got, want), "act_bwd differs at %d elements" % int((got != want).sum())
        x = rng.normal(size=n).astype(np.float32)
        xd = _cuda(x)
        yb, yv, yh = _buf(y)
        a = 0.2 + alpha
        rc, k = _launches(lambda: lib.cape_axpy(_p(yv), _p(xd), a, n, _st()))
        assert rc == 0 and k == 1
        _guard_ok(yb, yh, what="axpy")
        e = _rel(yv.cpu().numpy(), float(np.float32(a)) * x.astype(np.float64) + y)
        assert e <= 1e-6, e
        _report("act_bwd / axpy n=%d alpha=%g" % (n, alpha), e)


@pytest.mark.parametrize("row_floats,off,n", [(64, 0, 300), (7, 0, 300), (64, 1, 300), (20, 0, 300), (4, 0, 65535),
                                              (3, 0, 65535), (6890 * 3, 0, 40)])
def test_gather_rows(row_floats, off, n):
    """dst[i] = src[clamp(idx[i])]: the float4 path and the scalar path (rows not a multiple of 4 floats, or dst off
    16-byte alignment), repeated and out-of-range indices, n = 65535 rows.  Exact."""
    lib = _lib()
    rng = np.random.RandomState(row_floats + n)
    n_src = 97
    src = rng.normal(size=(n_src, row_floats)).astype(np.float32)
    idx = rng.randint(0, n_src, size=n).astype(np.int32)
    idx[:4] = [-5, n_src + 3, 0, n_src - 1]
    idx[4:8] = idx[8]
    want = src[np.clip(idx, 0, n_src - 1)]
    sd, idd = _cuda(src), _cuda(idx)
    db, d, dh = _buf(np.full(want.shape, NAN), head=off)
    rc, k = _launches(lambda: lib.cape_gather_rows(_p(sd), row_floats, n_src, _p(idd), n, _p(d), _st()))
    assert rc == 0 and k == 1
    _guard_ok(db, dh, head=off, what="gather")
    assert np.array_equal(d.cpu().numpy(), want)


def _wshapes():
    return [(Fin, K, Fout) for Fin in (1, 3, 35, 544) for K in (1, 2, 3, 6) for Fout in (1, 3, 35, 544)
            if Fin * Fout <= 35 * 544 or K <= 2]


@pytest.mark.parametrize("blocks", [1, 0])
def test_weight_prep(blocks):
    """Every descriptor of one launch: Fin, Fout of 1 / 3 / 35 / 544, K of 1 / 2 / 3 / 6, wt or wk NULL in some; the
    condition rows after the Fin K weight rows are NaN and must never reach an output.  Exact."""
    from cape_b200._lib import WPrep
    lib = _lib()
    rng = np.random.RandomState(blocks)
    shapes = _wshapes()
    keep, outs = [], []
    arr = (WPrep * len(shapes))()
    for i, (Fin, K, Fout) in enumerate(shapes):
        w = np.full((Fin * K + 5, Fout), NAN, np.float32)
        w[:Fin * K] = rng.normal(size=(Fin * K, Fout))
        wd = _cuda(w)
        w3 = w[:Fin * K].reshape(Fin, K, Fout)
        want_t = w3.transpose(1, 2, 0)                  # (k, c, f)
        want_k = w3.transpose(1, 0, 2)                  # (k, f, c)
        t = _buf(np.full(want_t.shape, NAN)) if i % 3 != 2 else None
        kk = _buf(np.full(want_k.shape, NAN)) if i % 3 != 1 else None
        d = arr[i]
        d.w, d.Fin, d.K, d.Fout = wd.data_ptr(), Fin, K, Fout
        d.wt = t[1].data_ptr() if t else None
        d.wk = kk[1].data_ptr() if kk else None
        keep.append(wd)
        outs.append((t, want_t, kk, want_k, (Fin, K, Fout)))
    table = _cuda(np.frombuffer(bytes(arr), dtype=np.uint8).copy())
    rc, k = _launches(lambda: lib.cape_weight_prep(_p(table), len(shapes), blocks, _st()))
    assert rc == 0 and k == 1
    for t, want_t, kk, want_k, shape in outs:
        for o, want, nm in ((t, want_t, "wt"), (kk, want_k, "wk")):
            if o is None:
                continue
            _guard_ok(o[0], o[2], what="%s %s" % (nm, shape))
            assert np.array_equal(o[1].cpu().numpy(), want), "%s %s" % (nm, shape)


def test_weight_transpose():
    """cape_cheb_weight_transpose: wt[c, k, f] = w[f, k, c] with NaN condition rows after the weights.  Exact."""
    lib = _lib()
    rng = np.random.RandomState(1)
    for (Fin, K, Fout) in _wshapes():
        w = np.full((Fin * K + 5, Fout), NAN, np.float32)
        w[:Fin * K] = rng.normal(size=(Fin * K, Fout))
        wd = _cuda(w)
        want = w[:Fin * K].reshape(Fin, K, Fout).transpose(2, 1, 0)
        tb, t, th = _buf(np.full(want.shape, NAN))
        rc, k = _launches(lambda: lib.cape_cheb_weight_transpose(_p(wd), Fin, K, Fout, _p(t), _st()))
        assert rc == 0 and k == 1
        _guard_ok(tb, th, what="wt %s" % ((Fin, K, Fout),))
        assert np.array_equal(t.cpu().numpy(), want), (Fin, K, Fout)


# ---------------------------------------------------------------------------------------------------------------------
# cape_gemm off its usual paths
# ---------------------------------------------------------------------------------------------------------------------
def gemm_case(case, M, N, K, ta, tb, *, tp=None, bias=False, act=0, alpha=0.5, beta=2.0, pad=0, launches=None,
              tol=None, seed=0):
    """C[:, :N] of an [M, N + pad] buffer = act(alpha A B + bias) + beta C against float64; the pad columns and the
    sentinels after C stay unchanged."""
    E = _E()
    tp = tp or _tp()
    rng = np.random.RandomState(seed + M + N + K)
    A = rng.normal(size=(K, M) if ta else (M, K)).astype(np.float32)
    B = rng.normal(size=(N, K) if tb else (K, N)).astype(np.float32)
    bv = rng.normal(size=N).astype(np.float32) if bias else None
    C0 = np.full((M, N + pad), NAN, np.float32)
    C0[:, :N] = rng.normal(size=(M, N))
    Am, Bm = (A.T if ta else A), (B.T if tb else B)
    want = alpha * (Am.astype(np.float64) @ Bm.astype(np.float64))
    if bias:
        want = want + bv
    if act == E.ACT_LEAKY:
        want = np.where(want > 0, want, E.LEAKY_ALPHA * want)
    elif act == E.ACT_RELU:
        want = np.maximum(want, 0)
    if beta:
        want = want + beta * C0[:, :N].astype(np.float64)
    Ad, Bd = _cuda(A), _cuda(B)
    cb, cv, ch = _buf(C0)
    _, n = _launches(lambda: E.gemm(tp, Ad.t() if ta else Ad, Bd.t() if tb else Bd, cv[:, :N],
                                    bias=_cuda(bv) if bias else None, act=act, alpha=alpha, beta=beta))
    if launches is not None:
        assert n == launches, (case, n, launches)
    got = cv.cpu().numpy()
    if pad:
        assert np.isnan(got[:, N:]).all(), "%s: wrote into the pad columns" % case
    _guard_ok(cb, ch, what=case)
    e = _rel(got[:, :N], want)
    tol = tol or (1e-5 if K <= 1000 else 1e-4)      # fp32 sums of 55168 products: ~1e-5 of max |C| is rounding
    _report(case, e)
    assert np.isfinite(got[:, :N]).all() and e <= tol, (case, e)
    return n


# the four operand layouts that otherwise take gemm_vec_kernel (FC forward / dW / dx shapes), on the scalar kernel
@pytest.mark.parametrize("M,N,K,ta,tb", [(5000, 64, 64, True, False), (4100, 64, 64, True, True),
                                         (64, 4100, 64, False, True), (1, 55168, 64, False, False)])
def test_gemm_scalar_kernel(M, N, K, ta, tb):
    with _knobs([(16, 1)]):
        gemm_case("gemm scalar M%d N%d K%d ta%d tb%d" % (M, N, K, ta, tb), M, N, K, ta, tb, bias=True,
                  act=_E().ACT_LEAKY)


def test_gemm_split_k_workspace():
    """The encoder-FC shape wants ~200 K splits: a handle without workspace runs it unsplit (one launch), one whose
    workspace holds 5 partial products runs 5 splits (+ the reduction); beta != 0 and ReLU through the reduction."""
    E = _E()
    M, N, K = 64, 128, 55168
    per = M * N * 4
    tp0 = E.Topology(0)
    gemm_case("gemm no workspace (unsplit)", M, N, K, False, False, tp=tp0, bias=True, launches=1)
    tp5 = E.Topology(0)
    tp5.reserve_workspace(5 * per + 100)
    gemm_case("gemm workspace for 5 splits", M, N, K, False, False, tp=tp5, bias=True, act=E.ACT_RELU, launches=2)
    gemm_case("gemm split-K beta=2", M, N, K, False, False, beta=2.0, launches=2)
    gemm_case("gemm split-K beta=-1 relu pad", M, N, K, True, False, beta=-1.0, act=E.ACT_RELU, pad=5, launches=2)


@pytest.mark.parametrize("M,N,K,ta,tb,pad", [(7, 3, 2, False, False, 3), (300, 130, 64, True, False, 7),
                                             (65, 66, 1000, False, True, 1), (5000, 64, 64, True, False, 4)])
def test_gemm_relu_wide_c(M, N, K, ta, tb, pad):
    """CAPE_ACT_RELU and a C inside a wider row (c_rs > N): the pad columns must stay unchanged."""
    gemm_case("gemm relu c_rs=N+%d M%d N%d K%d" % (pad, M, N, K), M, N, K, ta, tb, act=_E().ACT_RELU, bias=True,
              pad=pad)
