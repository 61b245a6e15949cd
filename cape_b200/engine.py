"""Thin Python layer over the C ABI: topology handle, conv sites, kernel-call helpers.

PyTorch is used only as plumbing (device buffers, streams); every compute call goes to libcape_b200.so.
"""
import ctypes as C

import numpy as np
import scipy.sparse as sp
import torch

from . import _lib
from . import topology as topo
from ._lib import (ACT_LEAKY, ACT_NONE, ACT_RELU, ACT_TANH, EPI_AFFINE, EPI_DUALMASK, EPI_LINEAR, EPI_SLOPE,
                   EPI_TANHGRAD, RECON_HUBER, RECON_L1, RECON_L2, ApplyArgs, ConvArgs, DwArgs, GemmItem, WPrep, check)

LEAKY_ALPHA = 0.2  # tf.nn.leaky_relu default (lib/models.py:109,506,582)

# The reference's `--activation` (self.brelu, lib/models.py:60,105-121) as (forward activation of the conv epilogue,
# data-gradient epilogue given the layer's output, its alpha).  ReLU's backward is the SLOPE mask with alpha 0: aux > 0
# on the output gives gradient 0 where the output is exactly 0, as tf.nn.relu's gradient does.
BRELU = {"b1leakyrelu": (ACT_LEAKY, EPI_SLOPE, LEAKY_ALPHA), "b1relu": (ACT_RELU, EPI_SLOPE, 0.0),
         "b1tanh": (ACT_TANH, EPI_TANHGRAD, 0.0)}
HUBER_DELTA = 0.1  # tf.losses.huber_loss(delta=0.1), lib/models.py:362-365


def recon_kind(loss):
    """The reconstruction loss of the reference's `--loss` (lib/models.py:357-369): 'l1' absolute difference, 'huber'
    Huber with delta 0.1, any other string the mean squared error."""
    return {"l1": RECON_L1, "huber": RECON_HUBER}.get(loss, RECON_L2)


def brelu(activation):
    """BRELU[activation]; the encoder / discriminator activations the reference defines but this port does not build
    raise here."""
    if activation not in BRELU:
        raise NotImplementedError("activation must be one of %s (lib/models.py:105-121); %r is not built"
                                  % (sorted(BRELU), activation))
    return BRELU[activation]

# Optional per-launch timing (bench.py's roofline pass): when PROFILE is a list, every helper below brackets its
# launch with CUDA events on the launching stream and appends (family, tag, algorithmic_bytes, ev0, ev1).
PROFILE = None
TRACE = bool(int(__import__("os").environ.get("CAPE_TRACE", "0")))   # debug: print and sync every conv launch


class _Prof:
    def __init__(self, family, tag):
        self.on = PROFILE is not None and tag is not None
        self.family, self.tag = family, tag

    def __enter__(self):
        if self.on:
            self.e0 = torch.cuda.Event(enable_timing=True)
            self.e1 = torch.cuda.Event(enable_timing=True)
            self.e0.record()
        return self

    def __exit__(self, *exc):
        if self.on:
            self.e1.record()
            PROFILE.append((self.family, self.tag[0], self.tag[1], self.e0, self.e1))
        return False


def _ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _f32(t):
    assert t.dtype == torch.float32 and t.is_cuda, "expected a CUDA fp32 tensor"
    return t


class Topology:
    """Owns a cape_topology handle on one device and the operator ids registered in it."""

    def __init__(self, device=0):
        self.lib = _lib.load()
        if not torch.cuda.is_available():
            raise _lib.CapeError("cape_b200 needs a CUDA device: there is no CPU execution path")
        self.device = torch.device("cuda", device if isinstance(device, int) else device.index or 0)
        h = C.c_void_p()
        check(self.lib.cape_topology_create(self.device.index, C.byref(h)))
        self.h = h
        self.op_shapes = []
        self._ws = 0

    def __del__(self):
        try:
            if getattr(self, "h", None):
                self.lib.cape_topology_destroy(self.h)
                self.h = None
        except Exception:
            pass

    def add_operator(self, m):
        """Register a scipy sparse matrix; returns its operator id."""
        idx, w = topo.to_ell(m)
        idx = np.ascontiguousarray(idx)
        w = np.ascontiguousarray(w)
        op = check(self.lib.cape_topology_add_operator(self.h, m.shape[0], m.shape[1], idx.shape[1],
                                                       idx.ctypes.data_as(C.c_void_p), w.ctypes.data_as(C.c_void_p)))
        self.op_shapes.append((m.shape[0], m.shape[1], idx.shape[1]))
        return op

    def reserve_workspace(self, nbytes):
        if nbytes > self._ws:
            check(self.lib.cape_topology_reserve_workspace(self.h, int(nbytes)))
            self._ws = int(nbytes)


class ConvSite:
    """One Chebyshev-conv call site: op_k = D . T_k(L~) . U for k < K (and the transposes for backward).

    Mirrors the operand triple the reference passes around: the Laplacian given to `filter`
    (lib/models.py:164,551,588,612,676,784,803), the U applied just before (:750,:782) and the D applied
    just after (:168,:807).
    """

    def __init__(self, tp, L, K, U=None, D=None, order_in=None, order_out=None):
        """order_in / order_out: internal vertex order (order[new] = reference index) of the level the site reads
        from / writes to; None = the reference's own numbering (topology.patch_order)."""
        self.K = K
        self.order_in, self.order_out = order_in, order_out
        self.ref_unpool, self.ref_pool = U is not None, D is not None   # poolwT calls in the reference graph
        self.M = L.shape[0]
        self.ref_rows_in = U.shape[1] if U is not None else L.shape[0]
        self.ref_rows_out = D.shape[0] if D is not None else L.shape[0]
        self.nnz = int(topo.rescale_L(L).nnz)
        # The reference computes pool(act(conv + b)) (lib/models.py:164-168); folding D into the operators computes
        # act(pool(conv) + b), which is the same only if D selects rows.  Callers that fuse a bias / activation check this.
        self.pool_is_selection = D is None or topo.is_selection(D)
        if U is not None and topo.is_identity(U, tol=1e-6):
            U = None     # factor-1 levels: identity up to 5e-11 (SURVEY.md section 0)
        if D is not None and topo.is_identity(D, tol=0):
            D = None
        T = topo.cheb_polynomials(L, K)
        self.rows_out = D.shape[0] if D is not None else L.shape[0]
        self.rows_in = U.shape[1] if U is not None else L.shape[0]
        self.ops, self.opsT, self.mats = [], [], []
        for k in range(K):
            m = topo.compose(D, T[k], U)
            if order_in is not None or order_out is not None:
                m = topo.permute(m, order_out, order_in)
            self.mats.append(m)
            if m.shape[0] == m.shape[1] and topo.is_identity(m, tol=0):
                self.ops.append(-1)
                self.opsT.append(-1)
            else:
                self.ops.append(tp.add_operator(m))
                self.opsT.append(tp.add_operator(sp.csr_matrix(m.T)))


# ---------------------------------------------------------------------------------------------------
# kernel-call helpers
# ---------------------------------------------------------------------------------------------------
def gemm(tp, A, B, Cout, bias=None, act=ACT_NONE, alpha=1.0, beta=0.0, tag=None, epilogue=EPI_LINEAR,
         epi_alpha=LEAKY_ALPHA, aux=None):
    """Cout = act(alpha * A @ B + bias) + beta * Cout for 2-D (possibly transposed) views; then, with epilogue SLOPE or
    TANHGRAD, the data-gradient epilogue given `aux` (a tensor of Cout's shape, unit column stride): cape_gemm_ex."""
    M, N, K, a_rs, a_cs, b_rs, b_cs = _gemm_strides(A, B, Cout)
    with _Prof("gemm", tag):
        if epilogue == EPI_LINEAR:
            check(tp.lib.cape_gemm(tp.h, M, N, K, _ptr(_f32(A)), a_rs, a_cs, _ptr(_f32(B)), b_rs, b_cs,
                                   _ptr(_f32(Cout)), Cout.stride(0), _ptr(bias), act, LEAKY_ALPHA, alpha, beta,
                                   _stream()))
            return
        assert tuple(aux.shape) == (M, N) and (aux.stride(1) == 1 or N == 1)
        check(tp.lib.cape_gemm_ex(tp.h, M, N, K, _ptr(_f32(A)), a_rs, a_cs, _ptr(_f32(B)), b_rs, b_cs, _ptr(_f32(Cout)),
                                  Cout.stride(0), _ptr(bias), act, LEAKY_ALPHA, alpha, beta, epilogue, epi_alpha,
                                  _ptr(_f32(aux)), aux.stride(0), _stream()))


def cheb_call(tp, N, rows_out, ncols, terms, out, out2=None, cond=None, epilogue=EPI_LINEAR, act=ACT_NONE,
              alpha=LEAKY_ALPHA, bias=None, bias_per_row=False, aux=None, tag=None, plain_only=False, family="ellconv"):
    """terms: list of dicts(src, op, F, src_rows, src_stride, w, w_stride, w2, wc, wc2) with torch tensors.
    plain_only: the cape_conv_args field of the same name (TMA-fed kernel or error)."""
    a = ConvArgs()
    a.plain_only = 1 if plain_only else 0
    a.N, a.rows_out, a.ncols, a.nterms = N, rows_out, ncols, len(terms)
    for i, t in enumerate(terms):
        d = a.terms[i]
        d.src = t["src"].data_ptr()
        d.op = t["op"]
        d.F = t["F"]
        d.src_rows = t["src_rows"]
        d.src_stride = t["src_stride"]
        d.w_stride = t["w_stride"]
        d.w2_stride = t.get("w2_stride", 0)
        d.w = t["w"].data_ptr() if t.get("w") is not None else None
        for k in ("w2", "wc", "wc2", "wT", "w2T", "stash"):
            v = t.get(k)
            setattr(d, k, v.data_ptr() if v is not None else None)
        d.wT_stride = t.get("wT_stride", 0)
        d.w2T_stride = t.get("w2T_stride", 0)
        d.stash_stride = t.get("stash_stride", 0)
    if cond is not None:
        a.cond = cond.data_ptr()
        a.C = cond.shape[1]
        assert cond.is_contiguous()
    a.epilogue, a.act, a.alpha = epilogue, act, alpha
    a.bias = bias.data_ptr() if bias is not None else None
    a.bias_per_row = 1 if bias_per_row else 0
    a.aux = aux.data_ptr() if aux is not None else None
    a.out = out.data_ptr()
    a.out2 = out2.data_ptr() if out2 is not None else None
    if TRACE:
        print("cheb_fwd", tag[0] if tag else None, N, rows_out, ncols, [(t["op"], t["F"]) for t in terms], flush=True)
    with _Prof(family, tag):
        check(tp.lib.cape_cheb_fwd(tp.h, C.byref(a), _stream()))
    if TRACE:
        torch.cuda.synchronize()


def apply_call(tp, N, rows_out, ncols, terms, out, out2=None, out_stride=0, cond=None, epilogue=EPI_LINEAR,
               act=ACT_NONE, alpha=LEAKY_ALPHA, bias=None, bias_per_row=False, aux=None, tag=None, family="ellconv",
               term_stride=0):
    """cape_apply: terms = list of dicts(src, op, src_rows, src_stride, acc=0, scale=1.0, wc=None, wc_stride=0)."""
    a = ApplyArgs()
    a.N, a.rows_out, a.ncols, a.nterms = N, rows_out, ncols, len(terms)
    for i, t in enumerate(terms):
        d = a.terms[i]
        d.src, d.op, d.src_rows, d.src_stride = t["src"].data_ptr(), t["op"], t["src_rows"], t["src_stride"]
        d.acc, d.scale = t.get("acc", 0), t.get("scale", 1.0)
        wc = t.get("wc")
        d.wc = wc.data_ptr() if wc is not None else None
        d.wc_stride = t.get("wc_stride", 0)
    if cond is not None:
        a.cond, a.C = cond.data_ptr(), cond.shape[1]
        assert cond.is_contiguous()
    a.epilogue, a.act, a.alpha = epilogue, act, alpha
    a.bias = bias.data_ptr() if bias is not None else None
    a.bias_per_row = 1 if bias_per_row else 0
    a.aux = aux.data_ptr() if aux is not None else None
    a.out, a.out_stride = out.data_ptr(), out_stride
    a.out2 = out2.data_ptr() if out2 is not None else None
    a.term_stride = term_stride
    if TRACE:
        print("apply", tag[0] if tag else None, N, rows_out, ncols, [(t["op"], t.get("scale", 1.0)) for t in terms], flush=True)
    with _Prof(family, tag):
        check(tp.lib.cape_apply(tp.h, C.byref(a), _stream()))
    if TRACE:
        torch.cuda.synchronize()


class WeightPrep:
    """All derived weight layouts of a network in ONE launch per optimiser step (cape_weight_prep): collect the layers'
    descriptors, upload the table once, then `run()` after every update."""

    def __init__(self, tp):
        self.tp, self.items, self.table = tp, [], None
        self.blocks_per_desc = int(__import__("os").environ.get("CAPE_WPREP_BLOCKS", "128"))

    def add(self, w, Fin, K, Fout, wt=None, wk=None):
        self.items.append((w, Fin, K, Fout, wt, wk))

    def run(self):
        if not self.items:
            return
        if self.table is None:
            arr = (WPrep * len(self.items))()
            for d, (w, Fin, K, Fout, wt, wk) in zip(arr, self.items):
                d.w, d.Fin, d.K, d.Fout = w.data_ptr(), Fin, K, Fout
                for nm, t in (("wt", wt), ("wk", wk)):
                    setattr(d, nm, t.data_ptr() if t is not None else None)
            raw = np.frombuffer(bytes(arr), dtype=np.uint8).copy()
            self.table = torch.from_numpy(raw).to(self.tp.device)
            torch.cuda.synchronize()
        # blocks per descriptor: the widest layer (512 x 2 x 512: 512 tiles of 32 x 32) sets the length of the launch,
        # blocks beyond a descriptor's tile count exit at once
        check(self.tp.lib.cape_weight_prep(C.c_void_p(self.table.data_ptr()), len(self.items), self.blocks_per_desc,
                                           _stream()))


def _gemm_strides(A, B, Cout):
    M, K = A.shape
    K2, N = B.shape
    assert K == K2 and tuple(Cout.shape) == (M, N) and (Cout.stride(1) == 1 or N == 1)
    a_rs, a_cs = A.stride()
    b_rs, b_cs = B.stride()
    if K == 1:          # degenerate dims: strides of size-1 axes are arbitrary in torch
        a_cs = 1
        if b_cs != 1:
            b_rs = 1
    if M == 1 and a_cs != 1:
        a_rs = 1
    if N == 1 and b_rs != 1:
        b_cs = 1
    return M, N, K, a_rs, a_cs, b_rs, b_cs


class SmallGemmBatch:
    """The tiny products of a training step (bias gradients, condition-channel gradients: ~80 per step, each a few
    microseconds of launch overhead) collected and issued as ONE launch (cape_gemm_batch).  `add` defers, `flush`
    launches; beta = 1 items accumulate atomically, so several may add into the same buffer.  The step's schedule is
    static: the device table of a schedule is built the first time it is seen (outside CUDA-graph capture)."""

    def __init__(self, tp):
        self.tp, self.pending, self.tables = tp, [], {}
        self.item_bytes = int(tp.lib.cape_gemm_item_bytes())
        self.blocks_per_item = int(__import__("os").environ.get("CAPE_SMALL_BLOCKS", "64"))

    def add(self, A, B, Cout, alpha=1.0, beta=0.0):
        M, N, K, a_rs, a_cs, b_rs, b_cs = _gemm_strides(A, B, Cout)
        self.pending.append((_f32(A).data_ptr(), a_rs, a_cs, _f32(B).data_ptr(), b_rs, b_cs, _f32(Cout).data_ptr(),
                             Cout.stride(0), M, N, K, float(alpha), float(beta)))

    def flush(self):
        if not self.pending:
            return
        key = tuple(self.pending)
        n = len(key)
        tab = self.tables.get(key)
        if tab is None:
            arr = (GemmItem * n)()
            for d, it in zip(arr, key):
                (d.a, d.a_rs, d.a_cs, d.b, d.b_rs, d.b_cs, d.c, d.c_rs, d.M, d.N, d.K, d.alpha, d.beta) = it
            tab = torch.empty(n * self.item_bytes, dtype=torch.uint8, device=self.tp.device)
            torch.cuda.synchronize()
            check(self.tp.lib.cape_gemm_batch(C.cast(arr, C.c_void_p), n, C.c_void_p(tab.data_ptr()), 0, _stream()))
            self.tables[key] = tab
        # blocks per item: the one wide product of a step (per-vertex output bias: [1 x N] @ [N x 20670], 323 column
        # tiles) sets the length of the launch; blocks beyond an item's tile count exit at once
        check(self.tp.lib.cape_gemm_batch(None, n, C.c_void_p(tab.data_ptr()), self.blocks_per_item, _stream()))
        self.pending = []


def tensor_cores_enabled(tp):
    return bool(tp.lib.cape_tensor_cores_enabled())


def cheb_dw(tp, N, rows_out, ncols, src, op, F, src_rows, src_stride, g, dw, dw_stride, accumulate=False, tag=None,
            dw_term_stride=0, dw_col_stride=0):
    """op: one operator id, or a list of them (all terms of a layer, term j written to dw + j * dw_term_stride)."""
    a = DwArgs()
    a.N, a.rows_out, a.ncols = N, rows_out, ncols
    if isinstance(op, (list, tuple)):
        a.nops, a.dw_term_stride, a.dw_col_stride = len(op), dw_term_stride, dw_col_stride
        for j, o in enumerate(op):
            a.ops[j] = o
        op = op[0]
    a.src, a.op, a.F, a.src_rows, a.src_stride = src.data_ptr(), op, F, src_rows, src_stride
    a.g, a.dw, a.dw_stride, a.accumulate = g.data_ptr(), dw.data_ptr(), dw_stride, 1 if accumulate else 0
    with _Prof("ellconv_dw", tag):
        check(tp.lib.cape_cheb_dw(tp.h, C.byref(a), _stream()))


def colsum(tp, g, N, rows, ncols, ops, out, g_stride=None):
    arr = (C.c_int * len(ops))(*ops)
    check(tp.lib.cape_colsum(tp.h, _ptr(g), ncols if g_stride is None else g_stride, N, rows, ncols, arr, len(ops),
                             _ptr(out), _stream()))


def weight_transpose(tp, w, Fin, K, Fout, wt):
    check(tp.lib.cape_cheb_weight_transpose(_ptr(w), Fin, K, Fout, _ptr(wt), _stream()))


def act_bwd(tp, dy, y, g, alpha=LEAKY_ALPHA):
    check(tp.lib.cape_act_bwd(_ptr(dy), _ptr(y), _ptr(g), dy.numel(), alpha, _stream()))


def axpy(tp, y, x, a):
    check(tp.lib.cape_axpy(_ptr(y), _ptr(x), float(a), y.numel(), _stream()))


def resample(tp, op, x, y, N, rows_out, rows_in, F, x_stride=None, y_stride=None, cond=None):
    check(tp.lib.cape_resample(tp.h, op, _ptr(x), F if x_stride is None else x_stride, _ptr(y),
                               F if y_stride is None else y_stride, N, rows_out, rows_in, F, _ptr(cond),
                               cond.shape[1] if cond is not None else 0, _stream()))


class SmplPoser:
    """Owns a cape_smpl handle: an SMPL body model resident on one device that poses batches of meshes [N, V, 3] with
    poses [N, 72] (cape_smpl_pose; the scratch is a torch buffer kept between calls)."""

    def __init__(self, jreg_ptr, jreg_col, jreg_val, posedirs, weights, parents, device=0):
        self.lib = _lib.load()
        if not torch.cuda.is_available():
            raise _lib.CapeError("cape_b200 needs a CUDA device: there is no CPU execution path")
        self.device = torch.device("cuda", device if isinstance(device, int) else device.index or 0)
        self.V = int(weights.shape[0])
        host = [np.ascontiguousarray(jreg_ptr, np.int32), np.ascontiguousarray(jreg_col, np.int32),
                np.ascontiguousarray(jreg_val, np.float32), np.ascontiguousarray(posedirs, np.float32),
                np.ascontiguousarray(weights, np.float32), np.ascontiguousarray(parents, np.int32)]
        h = C.c_void_p()
        check(self.lib.cape_smpl_create(self.device.index, self.V, *[a.ctypes.data_as(C.c_void_p) for a in host],
                                        C.byref(h)))
        self.h = h
        self.ws = torch.empty(0, dtype=torch.uint8, device=self.device)

    def __del__(self):
        try:
            if getattr(self, "h", None):
                self.lib.cape_smpl_destroy(self.h)
                self.h = None
        except Exception:
            pass

    def pose(self, verts, pose, out):
        """out[n] = verts[n] posed with pose[n]; fp32 CUDA tensors [N, V, 3], [N, 72], [N, V, 3]."""
        N = verts.shape[0]
        assert verts.shape == (N, self.V, 3) and pose.shape == (N, 72) and out.shape == verts.shape
        assert verts.is_contiguous() and pose.is_contiguous() and out.is_contiguous()
        nbytes = check(self.lib.cape_smpl_workspace_bytes(self.h, N))
        if self.ws.numel() < nbytes:
            self.ws = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
        check(self.lib.cape_smpl_pose(self.h, N, _ptr(_f32(verts)), _ptr(_f32(pose)), _ptr(_f32(out)), _ptr(self.ws),
                                      self.ws.numel(), _stream()))


def gn_relu_fwd(tp, x, gamma, beta, y, stats, G, eps=1e-5):
    N, rows, Cc = x.shape
    check(tp.lib.cape_gn_relu_fwd(tp.h, _ptr(x), N, rows, Cc, G, eps, _ptr(gamma), _ptr(beta), _ptr(y), _ptr(stats),
                                  _stream()))


def gn_relu_bwd(tp, x, y, dy, gamma, stats, dx, dgamma, dbeta, G, accumulate_dx=False):
    N, rows, Cc = x.shape
    check(tp.lib.cape_gn_relu_bwd(tp.h, _ptr(x), _ptr(y), _ptr(dy), N, rows, Cc, G, _ptr(gamma), _ptr(stats), _ptr(dx),
                                  1 if accumulate_dx else 0, _ptr(dgamma), _ptr(dbeta), _stream()))
