"""The reference's operator seam on top of the CUDA kernels.

The reference resolves its ops by name on `base_model` (lib/models.py:16-17,58-62):
filter='chebyshev5', pool/unpool='poolwT', activation='b1leakyrelu'.  The functions below keep those
names and argument meanings (x: [N, M, Fin] fp32, L / S: scipy sparse) but take the weights explicitly
instead of creating TF variables (b1leakyrelu exists only as chebyshev5's fused epilogue), and are differentiable through torch.autograd so a parity test reads
like a test of the reference op.  `chebyshev5` additionally exposes the fusions the kernels offer
(bias + activation, pooling D and unpooling U folded into the gather).
"""
import torch

from . import engine as E
from .engine import ACT_LEAKY, ACT_NONE, ACT_RELU, EPI_LINEAR, EPI_SLOPE, ConvSite, Topology

_topologies = {}
_sites = {}


def topology_for(device):
    idx = device.index if device.index is not None else torch.cuda.current_device()
    if idx not in _topologies:
        tp = Topology(idx)
        tp.reserve_workspace(64 << 20)
        _topologies[idx] = tp
    return _topologies[idx]


def _site(tp, L, K, U, D):
    key = (tp.device.index, id(L), K, id(U), id(D))
    if key not in _sites:
        _sites[key] = (ConvSite(tp, L, K, U=U, D=D), L, U, D)   # keep the matrices alive: ids stay unique
    return _sites[key][0]


class _ChebFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, W, bias, site, tp, act):
        N, M, Fin = x.shape
        K = site.K
        Fout = W.shape[1]
        x = x.contiguous()
        W = W.contiguous()
        out = torch.empty(N, site.rows_out, Fout, device=x.device)
        W3 = W.view(Fin, K, Fout)
        Wt = torch.empty(Fout, K, Fin, device=x.device)
        E.weight_transpose(tp, W, Fin, K, Fout, Wt)
        terms = [dict(src=x, op=site.ops[k], F=Fin, src_rows=site.rows_in, src_stride=Fin, w=W3[:, k, :],
                      w_stride=K * Fout, wT=Wt[:, k, :], wT_stride=K * Fin) for k in range(K)]
        b = bias.contiguous().view(-1) if bias is not None else None
        # one bias per filter ([F] / [1, 1, F]: b1*) or per vertex and filter ([1, M, F]: b2relu, lib/models.py:123-127)
        per_row = b is not None and b.numel() == site.rows_out * Fout and site.rows_out > 1
        assert b is None or per_row or b.numel() == Fout, "bias must be [F], [1, 1, F] or [1, M, F]"
        E.cheb_call(tp, N, site.rows_out, Fout, terms, out, epilogue=EPI_LINEAR, act=act, bias=b, bias_per_row=per_row)
        ctx.save_for_backward(x, W, out)
        ctx.site, ctx.tp, ctx.act, ctx.has_bias, ctx.per_row = site, tp, act, bias is not None, per_row
        ctx.bias_shape = tuple(bias.shape) if bias is not None else None
        return out

    @staticmethod
    def backward(ctx, dy):
        x, W, out = ctx.saved_tensors
        site, tp, act = ctx.site, ctx.tp, ctx.act
        N, _, Fin = x.shape
        K, Fout = site.K, W.shape[1]
        dy = dy.contiguous()
        if act == ACT_NONE:
            g = dy
        else:
            g = torch.empty_like(dy)
            E.act_bwd(tp, dy, out, g, alpha=E.LEAKY_ALPHA if act == ACT_LEAKY else 0.0)
        dW = torch.empty_like(W)
        dW3 = dW.view(Fin, K, Fout)
        for k in range(K):
            E.cheb_dw(tp, N, site.rows_out, Fout, x, site.ops[k], Fin, site.rows_in, Fin, g, dW3[:, k, :], K * Fout)
        db = None
        if ctx.has_bias and ctx.per_row:
            db = g.sum(0).view(ctx.bias_shape)
        elif ctx.has_bias:
            cs = torch.zeros(N, 1, Fout, device=x.device)
            E.colsum(tp, g, N, site.rows_out, Fout, [-1], cs)
            db = cs.sum(0).view(ctx.bias_shape)
        dx = None
        if ctx.needs_input_grad[0]:
            Wt = torch.empty(Fout, K, Fin, device=x.device)
            E.weight_transpose(tp, W, Fin, K, Fout, Wt)
            dx = torch.empty_like(x)
            W3 = W.view(Fin, K, Fout)
            terms = [dict(src=g, op=site.opsT[k], F=Fout, src_rows=site.rows_out, src_stride=Fout, w=Wt[:, k, :],
                          w_stride=K * Fin, wT=W3[:, k, :], wT_stride=K * Fout) for k in range(K)]
            E.cheb_call(tp, N, site.rows_in, Fin, terms, dx)
        return dx, dW, db, None, None, None


def chebyshev5(x, L, W, K, bias=None, activation=None, pool=None, unpool=None):
    """Chebyshev graph convolution y = sum_k T_k(L~) x W[k::K] (lib/models.py:69-103); W is [Fin*K, Fout] with row
    index fin*K + k.  Optional fusions: `unpool` U applied to x first (models.py:750,782), `bias`+`activation`
    ('b1leakyrelu' | 'b1relu' | 'b2relu' (bias [1, M, Fout]) | 'b1tanh' | None, models.py:105-127) and `pool` D applied
    last (models.py:168)."""
    tp = topology_for(x.device)
    if activation == "b1tanh":
        # lib/models.py:111-115; unused by every shipped config: the bias rides in the conv's epilogue, the tanh is a
        # separate elementwise pass (and comes before the pooling, as in the reference)
        y = torch.tanh(chebyshev5(x, L, W, K, bias=bias, activation=None, unpool=unpool))
        return poolwT(y, pool) if pool is not None else y
    act = {None: ACT_NONE, "b1leakyrelu": ACT_LEAKY, "b1relu": ACT_RELU, "b2relu": ACT_RELU}[activation]
    if pool is not None and bias is not None and bias.numel() > W.shape[1]:
        # a per-vertex bias (b2relu) lives on the un-pooled vertices: conv + bias + activation first, then the pooling
        y = _ChebFn.apply(x, W, bias, _site(tp, L, K, unpool, None), tp, act)
        return poolwT(y, pool)
    if pool is not None and (bias is not None or act != ACT_NONE):
        from . import topology as topo
        if not topo.is_selection(pool):
            # pooling commutes with the pointwise bias/activation only for row selections (the reference's D): a
            # general sampling matrix is applied after them, as the reference does (lib/models.py:164-168)
            y = _ChebFn.apply(x, W, bias, _site(tp, L, K, unpool, None), tp, act)
            return poolwT(y, pool)
    site = _site(tp, L, K, unpool, pool)
    return _ChebFn.apply(x, W, bias, site, tp, act)


class _ResampleFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, ops, tp):
        op, opT, rows_out, rows_in = ops
        x = x.contiguous()
        N, M, F = x.shape
        y = torch.empty(N, rows_out, F, device=x.device)
        E.resample(tp, op, x, y, N, rows_out, rows_in, F)
        ctx.ops, ctx.tp = ops, tp
        return y

    @staticmethod
    def backward(ctx, dy):
        op, opT, rows_out, rows_in = ctx.ops
        dy = dy.contiguous()
        N, _, F = dy.shape
        dx = torch.empty(N, rows_in, F, device=dy.device)
        E.resample(ctx.tp, opT, dy, dx, N, rows_in, rows_out, F)
        return dx, None, None


_resamplers = {}


def poolwT(x, S):
    """Pool / unpool with a precomputed sampling matrix S [M', M] (lib/models.py:129-152)."""
    import scipy.sparse as sp
    tp = topology_for(x.device)
    key = (tp.device.index, id(S))
    if key not in _resamplers:
        m = sp.csr_matrix(S)
        _resamplers[key] = ((tp.add_operator(m), tp.add_operator(sp.csr_matrix(m.T)), m.shape[0], m.shape[1]), S)
    return _ResampleFn.apply(x, _resamplers[key][0], tp)


def cnp(x, L, D, W, bias, K, activation="b1leakyrelu"):
    """Convolution, non-linearity, pooling: `base_model.cnp` (lib/models.py:154-171) as ONE fused launch -- the
    down-sampling D (a row selection) is folded into the operator tables, bias and activation into the epilogue."""
    return chebyshev5(x, L, W, K, bias=bias, activation=activation, pool=D)


def udn(x, L, U, W, bias, K, activation="b1leakyrelu"):
    """Unpool, (de)convolution, non-linearity: `base_model.udn` (lib/models.py:173-191) as ONE fused launch -- the
    up-sampling U is folded into the operator tables (op_k = T_k(L~) U), bias and activation into the epilogue.
    L is the Laplacian of the FINER level (the reference passes Laplacian[-i-2] with Upsample_mtx[-i-1])."""
    return chebyshev5(x, L, W, K, bias=bias, activation=activation, unpool=U)
