"""Explicit forward/backward executor for the CAPE mesh-VAE-GAN on the fixed SMPL hierarchy.

This replaces the TF-1.13 graph built by CAPE.build_graph (lib/models.py:267-351): the network is
static, so forward and backward are spelled out layer by layer over preallocated device buffers and
every layer is one (or a few) calls into libcape_b200.so.  Names in comments refer to the reference:
encoder :514-561, decoder_cond_vert :564-617, res_block_affine :776-793, res_block_decoder :744-774,
discriminator :648-678, loss :354-416, training :419-474.
"""
import contextlib
import gc
import math
import os

import numpy as np
import torch

from . import _lib
from . import engine as E
from . import topology as topo
from .engine import (ACT_LEAKY, ACT_NONE, EPI_AFFINE, EPI_DUALMASK, EPI_LINEAR, EPI_SLOPE, ConvSite, Topology,
                     act_bwd, axpy, cheb_call, cheb_dw, colsum, gemm)
from .params import init_params, is_d_param, is_g_param, param_specs


# tf.train.AdamOptimizer defaults (TF 1.13; lib/models.py:450-451), as the float32 tensors TF turns them into: the
# update's (1 - beta2) is 1 - fl32(0.999) = 9.9998713e-4, not 1e-3
ADAM_BETA1, ADAM_BETA2, ADAM_EPS = float(np.float32(0.9)), float(np.float32(0.999)), 1e-8


def _pad4(n):
    return (n + 3) // 4 * 4


class ParamStore:
    """Flat fp32 parameter / gradient / momentum buffers with named views (one all-reduce, one fused update)."""

    def __init__(self, specs, names, device):
        self.names = list(names)
        self.shapes = {n: tuple(specs[n]) for n in self.names}
        self.offsets = {}
        off = 0
        for n in self.names:
            self.offsets[n] = off
            off += _pad4(int(np.prod(self.shapes[n])))
        self.size = max(off, 4)
        self.flat = torch.zeros(self.size, device=device)
        self.grad = torch.zeros(self.size, device=device)
        self.mom = torch.zeros(self.size, device=device)
        self.lo = torch.zeros(self.size, device=device)     # flat - tf32_trunc(flat): cape_term.wT_lo (unread by the wgmma kernels)
        self.var = None                                     # Adam's second-moment slot (`mom` is its first): add_adam_slot()

    def add_adam_slot(self):
        if self.var is None:
            self.var = torch.zeros(self.size, device=self.flat.device)

    def lo_of(self, t):
        """The view of `lo` that corresponds to `t`, a contiguous view of `flat`; None if t is not one."""
        off = (t.data_ptr() - self.flat.data_ptr()) // 4
        if t.data_ptr() < self.flat.data_ptr() or off + t.numel() > self.size or not t.is_contiguous():
            return None
        return self.lo[off: off + t.numel()].view(t.shape)

    def _view(self, buf, n):
        k = int(np.prod(self.shapes[n]))
        return buf[self.offsets[n]: self.offsets[n] + k]

    def w(self, n):
        return self._view(self.flat, n)

    def g(self, n):
        return self._view(self.grad, n)

    def load(self, values):
        for n in self.names:
            self.w(n).copy_(torch.as_tensor(np.asarray(values[n], np.float32).reshape(-1)))

    def export(self, buf=None):
        buf = self.flat if buf is None else buf
        return {n: self._view(buf, n).detach().cpu().numpy().reshape(self.shapes[n]).copy() for n in self.names}


class Arena:
    """Bump allocator over one device buffer that is zeroed once per step (colsum targets)."""

    def __init__(self):
        self.reqs = []
        self.buf = None

    def request(self, *shape):
        self.reqs.append(shape)
        return len(self.reqs) - 1

    def build(self, device):
        offs, off = [], 0
        for s in self.reqs:
            offs.append(off)
            off += _pad4(int(np.prod(s)))
        self.buf = torch.zeros(max(off, 4), device=device)
        self.views = [self.buf[o: o + int(np.prod(s))].view(*s) for o, s in zip(offs, self.reqs)]

    def get(self, i):
        return self.views[i]

    def zero(self):
        self.buf.zero_()


def choose_dw_mode(F, Fout, K, rows_in, rows_out, need_dx, stash=True):
    """Where a layer's weight gradient takes its operands from (see ChebLayer): "aside" = basis stashed by the forward
    kernel, "gside" = op^T G stashed by the data-gradient kernel, "gather" = gathered again by cape_cheb_dw.
    The dense weight-gradient kernel needs F % 4 == 0, F >= 32 and 32 | Fout <= 512; pooled sites contract over the (fewer)
    output rows, un-pooling ones over the (fewer) input rows, same-level ones take the narrower side."""
    dense_ok = F % 4 == 0 and F >= 32 and Fout % 32 == 0 and Fout <= 512
    if not (dense_ok and stash):
        return "gather"
    if rows_out < rows_in:
        return "aside"
    if need_dx and (rows_in < rows_out or (K * Fout <= 512 and F >= Fout)):
        return "gside"
    return "aside"


def choose_forms(F, C, Fout, K, rows_in, rows_out, affine, need_dx, dw_mode, plain, name="", env=None):
    """(fwd_mode, dx_mode) of a conv layer -- how its forward / data-gradient pass is organised (the math is the same):
      "fused":    one kernel gathers the basis and contracts it (ellconv_tc.cu; thin layers: thin.cu);
      "basis":    cape_apply writes B_k = op_k x (forward: the stash the weight gradient reads anyway) or H_k = op_k^T G
                  (data gradient), then the tensor-core kernel contracts plain tensors;
      "contract": the tensor-core kernel computes Z = x @ [W_0 | W_1 | ..] (or G @ [W_k^T]_k) on the SOURCE rows, then
                  cape_apply applies the operators to the narrower Z and runs the epilogue.
    The defaults follow the work each form does; they have not been re-measured per layer on the H100:
      * forward: basis-first for the pooled K = 3 discriminator layers (the composed T_2 operator has ~19 taps, and the
        gathered basis is the stash the weight gradient reads anyway), contract-first for un-pooling layers (half the
        rows in the contraction, Fout-wide gathers), fused elsewhere;
      * data gradient: contract-first when the gradient narrows (Fout > F: the gathers run on the narrow side) or the
        layer pools and is at least 128 wide (the contraction runs on half the rows); basis-first for the wide
        un-pooling block only.
    Every tensor-core contraction accumulates in short per-chunk chains, so accuracy does not pick a form.
    Experiment overrides: CAPE_FWD_MODE / CAPE_DX_MODE for every layer, CAPE_MODES="enc/conv8:fwd=fused,disc/conv3:dx=contract"
    for single ones (ineligible requests are ignored).  `plain`: every operator of the site is the identity."""
    env = os.environ if env is None else env
    thin = F <= 4 or Fout <= 4
    split_ok = not thin and not plain and F % 16 == 0 and Fout % 16 == 0 and F >= 32 and Fout >= 32
    fwd_mode, dx_mode = "fused", "fused"
    basis_ok = C == 0 and not affine and dw_mode == "aside"
    if split_ok:
        if basis_ok and K >= 3 and rows_out < rows_in:
            # pooled K = 3 layers (the discriminator): the composed T_2 operator has ~19 taps, and the stash the fused kernel
            # writes next to its gather is what the separate gather launch produces anyway
            fwd_mode = "basis"
        elif (C > 0 or affine) and rows_in < rows_out:
            fwd_mode = "contract"
        # (an affine block has TWO upstream gradients -- d out and d out masked by the ReLU branch -- and the contract-first
        # data gradient projects only one tensor: fused for those.  No shipped config has an affine block that widens,
        # a generated 4-layer hierarchy does: tests/test_gpu_api.py::test_train_step_on_a_generated_4_layer_hierarchy)
        if (need_dx and not affine and dw_mode == "aside" and K * F <= 512
                and (Fout > F or (rows_out < rows_in and Fout == F and F >= 128))):
            dx_mode = "contract"
        if need_dx and dw_mode == "gside" and rows_in < rows_out and Fout >= 128:
            # wide un-pooling block (dec/aff3: 256 -> 128 at 862 -> 1723 rows): H = op^T G by the gather kernel into the
            # weight gradient's stash, then one plain contraction; the narrower un-pooling blocks stay fused
            dx_mode = "basis"
    fm, dm = env.get("CAPE_FWD_MODE", ""), env.get("CAPE_DX_MODE", "")
    for item in filter(None, env.get("CAPE_MODES", "").split(",")):
        key, val = item.split("=")
        if key == name + ":fwd":
            fm = val
        elif key == name + ":dx":
            dm = val
    if fm and (fm == "fused" or (split_ok and (fm != "basis" or basis_ok))):
        fwd_mode = fm
    if dm and need_dx and (dm == "fused" or (split_ok and (dm != "basis" or dw_mode == "gside")
                                             and (dm != "contract" or (dw_mode != "gside" and not affine)))):
        dx_mode = dm
    return fwd_mode, dx_mode


class ChebLayer:
    """chebyshev5 (+bias/act, +pool/unpool folded into the site, +condition channels, + optional affine
    branch) with its backward."""

    def __init__(self, net, site, F, C, Fout, W, gW, bias=None, gbias=None, act=ACT_NONE, Wa=None, gWa=None,
                 bias_per_row=False, need_dx=True, maxN=1, n_cs_slots=1, name="", fused=False):
        """fused: always the one-launch forms, so that a caller can add terms of its own to the launch (fwd / bwd
        `extra`)."""
        self.net, self.tp, self.site, self.name = net, net.tp, site, name
        if (bias is not None or act != ACT_NONE) and not site.pool_is_selection:
            raise NotImplementedError("%s: the down-sampling matrix is not a pure row selection, so pooling cannot be "
                                      "folded in front of the bias/activation (lib/models.py:164-168 applies them "
                                      "before the pool)" % name)
        self.F, self.C, self.Fout, self.K = F, C, Fout, site.K
        K = self.K
        self.W3, self.gW3 = W.view(F + C, K, Fout), gW.view(F + C, K, Fout)
        self.W, self.bias, self.gbias, self.act = W, bias, gbias, act
        self.bias_per_row = bias_per_row
        self.affine = Wa is not None
        if self.affine:
            self.Wa, self.Wa2, self.gWa2 = Wa, Wa.view(F + C, Fout), gWa.view(F + C, Fout)
        self.need_dx = need_dx
        dev = W.device
        # Derived weight layouts, refreshed after every update by ONE batched launch (net.wprep):
        #   Wt [K(+1), Fout, F]: per-order K-major copies (+ the affine branch as order K): B operand of the tensor-core
        #      forward, fp32-pipe operand of the data gradient; read as [(k, c), f] it is the B operand of the
        #      contract-first forward Z = X @ [W_0 | W_1 | ... | W_a];
        #   Wk [K, F, Fout]: per-order plain copies, B operand of the contract-first data gradient Z = G @ [W_k^T]_k.
        A = 1 if self.affine else 0
        self.Wt, self.Wt_lo = torch.empty(K + A, Fout, F, device=dev), torch.empty(K + A, Fout, F, device=dev)
        self.W3_lo = net.lo_of(W).view(F + C, K, Fout)
        net.wprep.add(W, F, K, Fout, wt=self.Wt[:K], wt_lo=self.Wt_lo[:K])
        if self.affine:
            self.Wa2_lo = net.lo_of(Wa).view(F + C, Fout)
            net.wprep.add(Wa, F, 1, Fout, wt=self.Wt[K:], wt_lo=self.Wt_lo[K:])
        # Where the weight gradient gets its operands (all three end in the same contraction  dW = A^T G over rows):
        #   "aside":  the forward kernel also writes the gathered basis B_k = op_k x (cape_term.stash), dW_k = B_k^T G;
        #   "gside":  the data-gradient kernel also writes H_k = op_k^T G, dW_k = x^T H_k -- all K terms in ONE pass
        #             over x when K*Fout <= 512 (the widest weight-gradient tile set), over the smaller row set when the site un-pools;
        #   "gather": cape_cheb_dw gathers the basis again (thin layers, odd shapes).
        # The first two make both operands plain tensors, which the weight-gradient kernel reads without a gather.
        self.dw_mode = choose_dw_mode(F, Fout, K, site.rows_in, site.rows_out, need_dx,
                                      os.environ.get("CAPE_DW_STASH", "1") != "0")
        self.stash_a, self.stash_g, self.stash_ga = [None] * K, [None] * K, None
        if self.dw_mode == "aside":
            # the basis tensors of the non-identity terms, contiguous: cape_apply writes all of them in one launch
            nz = [k for k in range(K) if site.ops[k] != -1]
            self.stash_all = torch.empty(max(len(nz), 1), maxN, site.rows_out, F, device=dev)
            self.stash_a = [None] * K
            for j, k in enumerate(nz):
                self.stash_a[k] = self.stash_all[j]
        elif self.dw_mode == "gside":
            self.g_merged = K > 1 and K * Fout <= 512
            if self.g_merged:
                self.Hg = torch.empty(maxN, site.rows_in, K * Fout, device=dev)
                self.stash_g = [self.Hg[:, :, k * Fout:(k + 1) * Fout] for k in range(K)]
            else:
                self.stash_g = [None if site.opsT[k] == -1 else torch.empty(maxN, site.rows_in, Fout, device=dev)
                                for k in range(K)]
            if self.affine and site.opsT[0] != -1:
                self.stash_ga = torch.empty(maxN, site.rows_in, Fout, device=dev)
        self.fwd_mode, self.dx_mode = choose_forms(F, C, Fout, K, site.rows_in, site.rows_out, self.affine, need_dx,
                                                   self.dw_mode, all(o == -1 for o in site.ops), name)
        if fused:
            self.fwd_mode, self.dx_mode = "fused", "fused"
        if self.dx_mode == "contract":
            self.Wk, self.Wk_lo = torch.empty(K, F, Fout, device=dev), torch.empty(K, F, Fout, device=dev)
            net.wprep.add(W, F, K, Fout, wk=self.Wk, wk_lo=self.Wk_lo)
            net.scratch_req(maxN * site.rows_out * K * F)
        if self.fwd_mode == "contract":
            net.scratch_req(maxN * site.rows_in * (K + A) * Fout)
        # colsum targets: [bias?] + K condition sums (+1 for the affine branch)
        self.cs_ops = []
        if bias is not None and not bias_per_row:
            self.cs_ops.append(-1)
        self.cs_cond0 = len(self.cs_ops)
        if C:
            self.cs_ops += list(site.ops)
        # one zero-initialised target per backward call made within a step (colsum accumulates atomically)
        self.cs_id = [net.arena.request(maxN, max(len(self.cs_ops), 1), Fout) for _ in range(n_cs_slots)]
        self.csa_id = net.arena.request(maxN, 1, Fout) if (self.affine and C) else None

    def alg_bytes(self, N, what):
        """Algorithmic bytes of what this layer's launches replace in the reference graph, per SURVEY.md 8(d):
        every tensor crossing a layer boundary once, fp32, Fin INCLUDING the materialised condition channels;
        conv fwd 4NM(Fin+Fout) + 4*Fin*K*Fout (+12 nnz if K>1), resample 4NF(M+M'), bwd = 4NM(2Fin+Fout) + 2x weights
        (attributed: dx launch = Fin+Fout share + resamples, dW launches = the extra Fin share)."""
        s, Fin, Fo, K = self.site, self.F + self.C, self.Fout, self.K
        wbytes = 4 * Fin * K * Fo + (12 * s.nnz if K > 1 else 0)
        conv = 4 * N * s.M * (Fin + Fo) + wbytes
        if self.affine:
            conv += 4 * N * s.M * (Fin + Fo) + 4 * Fin * Fo
            wbytes += 4 * Fin * Fo
        res = 0
        if s.ref_unpool:
            res += 4 * N * Fin * (s.ref_rows_in + s.M)
        if s.ref_pool:
            res += 4 * N * Fo * (s.M + s.ref_rows_out)
        if what in ("fwd", "dx"):
            return conv + res
        return 4 * N * s.M * Fin * (2 if self.affine else 1) + wbytes      # all dW launches of the layer together

    def _split(self):
        """The split forms need the tensor-core kernels (they pass K-major weights only)."""
        return E.tensor_cores_enabled(self.tp)

    def fwd(self, x, ycat, out, out2=None, extra=()):
        """extra: more cheb_call terms of the same launch (a layer built with fused=True)."""
        N = x.shape[0]
        s, F, C, K, Fout = self.site, self.F, self.C, self.K, self.Fout
        assert x.shape[1] == s.rows_in and x.shape[2] >= F and out.shape[1] == s.rows_out
        sx = x.shape[2]
        tag = (self.name + ":fwd", self.alg_bytes(N, "fwd"))
        sub = lambda what: (self.name + ":fwd/" + what, 0)           # bytes are booked on the layer's main launch
        if self.fwd_mode == "contract" and self._split():
            A = 1 if self.affine else 0
            ncz = (K + A) * Fout
            Z = self.net.scratch[: N * s.rows_in * ncz].view(N, s.rows_in, ncz)
            cheb_call(self.tp, N, s.rows_in, ncz,
                      [dict(src=x, op=-1, F=F, src_rows=s.rows_in, src_stride=sx, w=None, w_stride=0,
                            wT=self.Wt.view(ncz, F), wT_stride=F, wT_lo=self.Wt_lo.view(ncz, F))],
                      Z, plain_only=True, tag=sub("project"))
            terms = [dict(src=Z[:, :, k * Fout:], op=s.ops[k], src_rows=s.rows_in, src_stride=ncz, acc=0,
                          wc=self.W3[F:, k, :] if C else None, wc_stride=K * Fout) for k in range(K)]
            if self.affine:
                terms.append(dict(src=Z[:, :, K * Fout:], op=s.ops[0], src_rows=s.rows_in, src_stride=ncz, acc=1,
                                  wc=self.Wa2[F:] if C else None, wc_stride=Fout))
            E.apply_call(self.tp, N, s.rows_out, Fout, terms, out, out2=out2, cond=ycat if C else None,
                         epilogue=EPI_AFFINE if self.affine else EPI_LINEAR, act=self.act, bias=self.bias,
                         bias_per_row=self.bias_per_row, tag=tag)
            return
        basis = self.fwd_mode == "basis" and self._split()
        if basis:
            # B_k = op_k x for every non-identity term by ONE gather launch, written where the weight gradient reads them
            nz = [k for k in range(K) if s.ops[k] != -1]
            if N == self.stash_all.shape[1]:
                E.apply_call(self.tp, N, s.rows_out, F, [dict(src=x, op=s.ops[k], src_rows=s.rows_in, src_stride=sx) for k in nz],
                             self.stash_all, term_stride=self.stash_all.stride(0), tag=sub("basis"))
            else:                                   # a partial batch: the tensors of the terms are not adjacent then
                for k in nz:
                    E.apply_call(self.tp, N, s.rows_out, F, [dict(src=x, op=s.ops[k], src_rows=s.rows_in, src_stride=sx)],
                                 self.stash_a[k][:N], tag=sub("basis%d" % k))
        terms = []
        for k in range(K):
            t = dict(src=x, op=s.ops[k], F=F, src_rows=s.rows_in, src_stride=sx, w=self.W3[:, k, :],
                     w_stride=K * Fout, wT=self.Wt[k], wT_stride=F, wT_lo=self.Wt_lo[k])
            if C:
                t["wc"] = self.W3[F:, k, :]
            if basis and s.ops[k] != -1:
                t.update(src=self.stash_a[k][:N], op=-1, src_rows=s.rows_out, src_stride=F)   # contracted as a plain tensor
            elif self.stash_a[k] is not None:
                t["stash"], t["stash_stride"] = self.stash_a[k][:N], F
            if self.affine and k == 0:
                t["w2"], t["w2_stride"] = self.Wa2, Fout
                t["w2T"], t["w2T_stride"], t["w2T_lo"] = self.Wt[K], F, self.Wt_lo[K]
                if C:
                    t["wc2"] = self.Wa2[F:]
            terms.append(t)
        cheb_call(self.tp, N, s.rows_out, Fout, terms + list(extra), out, out2=out2, cond=ycat if C else None,
                  epilogue=EPI_AFFINE if self.affine else EPI_LINEAR, act=self.act, bias=self.bias,
                  bias_per_row=self.bias_per_row, tag=tag)

    def bwd(self, x, ycat, g, g_aff=None, dx=None, dx2=None, dx_epi=EPI_LINEAR, dx_aux=None, dx_alpha=E.LEAKY_ALPHA,
            dycat=None, want_dw=True, cs_slot=0, dx_extra=()):
        """g: gradient w.r.t. the pre-activation of accumulator 0 ([N, rows_out, Fout]);
        g_aff: gradient w.r.t. the affine branch (= d out) when the layer has one;
        dx_extra: more terms of the data-gradient launch (a layer built with fused=True)."""
        tp, s, F, C, K, Fout = self.tp, self.site, self.F, self.C, self.K, self.Fout
        N = g.shape[0]
        sx = x.shape[2]
        mode = self.dw_mode if (want_dw and (self.dw_mode != "gside" or dx is not None)) else "gather"
        if want_dw and mode == "aside":
            nl = K + (1 if self.affine else 0)
            tg = (self.name + ":dW", self.alg_bytes(N, "dW") / nl)

            def dw_aside(tp):
                for k in range(K):
                    B = self.stash_a[k]
                    if B is None:                               # identity term: the basis is x itself
                        cheb_dw(tp, N, s.rows_out, Fout, x, -1, F, s.rows_in, sx, g, self.gW3[:, k, :], K * Fout, tag=tg)
                    else:
                        cheb_dw(tp, N, s.rows_out, Fout, B[:N], -1, F, s.rows_out, F, g, self.gW3[:, k, :], K * Fout,
                                tag=tg)
                if self.affine:
                    B = self.stash_a[0]
                    if B is None:
                        cheb_dw(tp, N, s.rows_out, Fout, x, -1, F, s.rows_in, sx, g_aff, self.gWa2, Fout, tag=tg)
                    else:
                        cheb_dw(tp, N, s.rows_out, Fout, B[:N], -1, F, s.rows_out, F, g_aff, self.gWa2, Fout, tag=tg)
            self.net.run_dw(dw_aside)
        elif (want_dw and mode == "gather" and Fout <= 4 and not self.affine and F in (32, 64, 128, 256) and sx == F
              and K <= 4):
            # thin OUTPUT: swap the roles -- operators on the narrow gradient (H_k = op_k^T g), one pass over x;
            # dW_k[f, c] = sum_r x[r, f] H_k[r, c] lands in the [F, K, Fout] layout through the three strides
            cheb_dw(tp, N, s.rows_in, F, g, list(s.opsT), Fout, s.rows_out, Fout, x, self.gW3, 1,
                    tag=(self.name + ":dW", self.alg_bytes(N, "dW")), dw_term_stride=Fout, dw_col_stride=K * Fout)
        elif want_dw and mode == "gather":
            nl = (1 if F <= 4 else K) + (1 if self.affine else 0)
            tg = (self.name + ":dW", self.alg_bytes(N, "dW") / nl)
            if F <= 4:          # thin input: all K terms in one pass over g
                cheb_dw(tp, N, s.rows_out, Fout, x, list(s.ops), F, s.rows_in, sx, g, self.gW3, K * Fout, tag=tg,
                        dw_term_stride=Fout)
            for k in range(K if F > 4 else 0):
                cheb_dw(tp, N, s.rows_out, Fout, x, s.ops[k], F, s.rows_in, sx, g, self.gW3[:, k, :], K * Fout, tag=tg)
            if self.affine:
                cheb_dw(tp, N, s.rows_out, Fout, x, s.ops[0], F, s.rows_in, sx, g_aff, self.gWa2, Fout, tag=tg)
        has_bias = self.bias is not None and not self.bias_per_row and want_dw
        if (has_bias or C) and len(self.cs_ops):
            cs = self.net.arena.get(self.cs_id[cs_slot])[:N]
            nops = len(self.cs_ops)
            if nops <= 4:
                # the column sums feed nothing but the deferred small products: next to the weight gradients on the side
                # stream (they read the same gradient tensor), always through the main handle (it owns the row sums)
                self.net.run_glue(lambda: colsum(tp, g, N, s.rows_out, Fout, self.cs_ops, cs))
            else:
                for o in range(0, nops, 4):
                    self._colsum_chunk(g, N, cs, o)
            sg = self.net.small.add                  # tiny products: deferred, one launch per step (SmallGemmBatch)
            if has_bias:
                sg(self.net.ones[:, :N], cs[:, 0, :], self.gbias.view(1, Fout))
            if C:
                for k in range(K):
                    dq = cs[:, self.cs_cond0 + k, :]
                    if want_dw:
                        sg(ycat.t(), dq, self.gW3[F:, k, :])
                    if dycat is not None:
                        sg(dq, self.W3[F:, k, :].t(), dycat, beta=1.0)
        if self.affine and C:
            csa = self.net.arena.get(self.csa_id)[:N]
            self.net.run_glue(lambda: colsum(tp, g_aff, N, s.rows_out, Fout, [s.ops[0]], csa))
            if want_dw:
                self.net.small.add(ycat.t(), csa[:, 0, :], self.gWa2[F:])
            if dycat is not None:
                self.net.small.add(csa[:, 0, :], self.Wa2[F:].t(), dycat, beta=1.0)
        if self.bias_per_row and want_dw:
            self.net.small.add(self.net.ones[:, :N], g.view(N, s.rows_out * Fout), self.gbias.view(1, s.rows_out * Fout))
        if dx is not None:
            assert self.need_dx
            gs = want_dw and mode == "gside"
            dtag = (self.name + ":dx", self.alg_bytes(N, "dx"))
            sub = lambda what: (self.name + ":dx/" + what, 0)
            if self.dx_mode == "contract" and self._split():
                # Z = G @ [W_0^T | W_1^T | ..] on the (pooled / narrower) output rows, then dX = epi(sum_k op_k^T Z_k)
                Z = self.net.scratch[: N * s.rows_out * K * F].view(N, s.rows_out, K * F)
                cheb_call(tp, N, s.rows_out, K * F,
                          [dict(src=g, op=-1, F=Fout, src_rows=s.rows_out, src_stride=Fout, w=None, w_stride=0,
                                wT=self.Wk.view(K * F, Fout), wT_stride=Fout, wT_lo=self.Wk_lo.view(K * F, Fout))],
                          Z, plain_only=True, tag=sub("project"))
                E.apply_call(tp, N, s.rows_in, F,
                             [dict(src=Z[:, :, k * F:], op=s.opsT[k], src_rows=s.rows_out, src_stride=K * F)
                              for k in range(K)], dx, out2=dx2, epilogue=dx_epi, aux=dx_aux, alpha=dx_alpha, tag=dtag)
            else:
                basis = gs and self.dx_mode == "basis" and self._split()
                terms = []
                if self.affine:
                    t = dict(src=g_aff, op=s.opsT[0], F=Fout, src_rows=s.rows_out, src_stride=Fout, w=self.Wt[K],
                             w_stride=F, wT=self.Wa2, wT_stride=Fout, wT_lo=self.Wa2_lo)
                    if gs and self.stash_ga is not None:
                        t["stash"], t["stash_stride"] = self.stash_ga[:N], Fout
                    terms.append(t)
                for k in range(K):
                    t = dict(src=g, op=s.opsT[k], F=Fout, src_rows=s.rows_out, src_stride=Fout,
                             w=self.Wt[k], w_stride=F, wT=self.W3[:, k, :], wT_stride=K * Fout,
                             wT_lo=self.W3_lo[:, k, :])
                    if gs and self.stash_g[k] is not None:
                        t["stash"], t["stash_stride"] = self.stash_g[k][:N], self.stash_g[k].stride(1)
                    terms.append(t)
                if basis:
                    # H = op^T G by the gather kernel into the buffers the weight gradient reads; contracted as plain tensors
                    for i, t in enumerate(terms):
                        if t["op"] == -1:
                            continue
                        H, hs = t.pop("stash"), t.pop("stash_stride")
                        E.apply_call(tp, N, s.rows_in, Fout,
                                     [dict(src=t["src"], op=t["op"], src_rows=s.rows_out, src_stride=Fout)], H,
                                     out_stride=hs, tag=sub("narrow%d" % i))
                        t.update(src=H, op=-1, src_rows=s.rows_in, src_stride=hs)
                cheb_call(tp, N, s.rows_in, F, terms + list(dx_extra), dx, out2=dx2, epilogue=dx_epi, aux=dx_aux,
                          alpha=dx_alpha, tag=dtag)
            if gs:
                # dW_k = x^T (op_k^T G): the data-gradient kernel above left op_k^T G in the stash buffers
                nl = (1 if self.g_merged else K) + (1 if self.affine else 0)
                tg = (self.name + ":dW", self.alg_bytes(N, "dW") / nl)

                def dw_gside(tp):
                    if self.g_merged:
                        cheb_dw(tp, N, s.rows_in, K * Fout, x, -1, F, s.rows_in, sx, self.Hg[:N], self.gW3, K * Fout, tag=tg)
                    else:
                        for k in range(K):
                            H = g if self.stash_g[k] is None else self.stash_g[k][:N]
                            cheb_dw(tp, N, s.rows_in, Fout, x, -1, F, s.rows_in, sx, H, self.gW3[:, k, :], K * Fout,
                                    tag=tg)
                    if self.affine:
                        Ha = g_aff if self.stash_ga is None else self.stash_ga[:N]
                        cheb_dw(tp, N, s.rows_in, Fout, x, -1, F, s.rows_in, sx, Ha, self.gWa2, Fout, tag=tg)
                self.net.run_dw(dw_gside)

    def _colsum_chunk(self, g, N, cs, o):
        # more than 4 operators (K > 3 with conditions): contiguous scratch per chunk, then copy back
        ops = self.cs_ops[o:o + 4]
        tmp = torch.zeros(N, len(ops), self.Fout, device=g.device)
        colsum(self.tp, g, N, self.site.rows_out, self.Fout, ops, tmp)
        cs[:, o:o + len(ops), :] = tmp


class Dense:
    """tf.layers.dense (y = act(xW + b)) with backward."""

    def __init__(self, net, W, b, gW, gb, act=ACT_NONE, name=""):
        self.net, self.tp, self.name = net, net.tp, name
        self.W, self.b, self.gW, self.gb, self.act = W, b, gW, gb, act

    def fwd(self, x, out):
        M, K = x.shape
        Nn = self.W.shape[1]
        gemm(self.tp, x, self.W, out, bias=self.b, act=self.act,
             tag=(self.name + ":fwd", 4 * (M * (K + Nn) + K * Nn)))      # SURVEY 8(d): 4N(in+out) + 4 in*out

    def bwd(self, x, out, dout, gtmp=None, dx=None, dx_beta=0.0, want_dw=True):
        g = dout
        if self.act != ACT_NONE:
            act_bwd(self.tp, dout, out, gtmp)
            g = gtmp
        N = g.shape[0]
        if want_dw:
            gemm(self.tp, x.t(), g, self.gW)
            gemm(self.tp, self.net.ones[:, :N], g, self.gb.view(1, -1))
        if dx is not None:
            gemm(self.tp, g, self.W.t(), dx, beta=dx_beta)


class GNBlock:
    """GraphCMR-style decoder residual block with group norm (res_block_decoder, lib/models.py:744-774):
    Z = unpool([x ; cond]); h = lin1(relu(GN(Z))); h = cheb_K(relu(GN(h))); out = lin2(relu(GN(h))) + lin_in(Z).
    The concat+unpool is one gather kernel (condition channels = rowsum(U) * y, never read from HBM), every
    GN+ReLU is one fused pass each way, lin2 + lin_in is a single two-term contraction."""

    def __init__(self, net, idx, L, U, Fin, Cc, Fo, K, scope, maxN, order_in=None, order_out=None):
        import scipy.sparse as sp
        self.net, self.tp = net, net.tp
        tp, dev = net.tp, net.device
        w, g = net._w, net._g
        self.Fin, self.Cc, self.Ft, self.mid, self.Fo = Fin, Cc, Fin + Cc, Fo // 2, Fo
        self.rows, self.rows_in = L.shape[0], U.shape[1]
        if topo.is_identity(U, tol=1e-6) and order_in is order_out:
            self.op_u = self.op_uT = -1
        else:
            Up = topo.permute(sp.identity(U.shape[0], format="csr") if topo.is_identity(U, tol=1e-6) else U,
                              order_out, order_in)
            self.op_u, self.op_uT = tp.add_operator(sp.csr_matrix(Up)), tp.add_operator(sp.csr_matrix(Up.T))
        lin = ConvSite(tp, L, 1, order_in=order_out, order_out=order_out)
        conv = ConvSite(tp, L, K, order_in=order_out, order_out=order_out)
        self.order_out = order_out
        nm = "dec/res%d" % (idx + 1)
        mk = lambda site, F, Fout, sc, tag: ChebLayer(net, site, F, 0, Fout, w(scope + "/" + sc + "/weights"),
                                                      g(scope + "/" + sc + "/weights"), maxN=maxN, name=nm + "/" + tag)
        self.lin1 = mk(lin, self.Ft, self.mid, "graph_linear_1", "lin1")
        self.conv = mk(conv, self.mid, self.mid, "graph_conv", "graph_conv")
        self.lin2 = mk(lin, self.mid, Fo, "graph_linear_2", "lin2")
        # the skip connection is projected only when the channel counts differ (lib/models.py:764-768)
        self.lin_in = (mk(lin, self.Ft, Fo, "graph_linear_input", "lin_in")
                       if (scope + "/graph_linear_input/weights") in net.specs else None)
        self.gn = []
        for sc, C in (("group_norm", self.Ft), ("group_norm_1", self.mid), ("group_norm_2", self.mid)):
            self.gn.append(dict(C=C, G=min(32, C), gamma=w(scope + "/" + sc + "/gamma"), beta=w(scope + "/" + sc + "/beta"),
                                dgamma=g(scope + "/" + sc + "/gamma"), dbeta=g(scope + "/" + sc + "/beta"),
                                stats=torch.zeros(maxN, min(32, C), 2, device=dev)))
        z = lambda *sh: torch.zeros(*sh, device=dev)
        N, M = maxN, self.rows
        self.Z, self.A1 = z(N, M, self.Ft), z(N, M, self.Ft)
        self.H1, self.A2, self.H2, self.A3 = z(N, M, self.mid), z(N, M, self.mid), z(N, M, self.mid), z(N, M, self.mid)
        self.dZ, self.dA1 = z(N, M, self.Ft), z(N, M, self.Ft)
        self.dH1, self.dA2, self.dH2, self.dA3 = z(N, M, self.mid), z(N, M, self.mid), z(N, M, self.mid), z(N, M, self.mid)

    def layers(self):
        return [l for l in (self.lin1, self.conv, self.lin2, self.lin_in) if l is not None]

    def fwd(self, x, ycat, out):
        tp, N = self.tp, x.shape[0]
        E.resample(tp, self.op_u, x, self.Z, N, self.rows, self.rows_in, self.Fin, x_stride=x.shape[2],
                   y_stride=self.Ft, cond=ycat)
        g0, g1, g2 = self.gn
        E.gn_relu_fwd(tp, self.Z, g0["gamma"], g0["beta"], self.A1, g0["stats"], g0["G"])
        self.lin1.fwd(self.A1, None, self.H1)
        E.gn_relu_fwd(tp, self.H1, g1["gamma"], g1["beta"], self.A2, g1["stats"], g1["G"])
        self.conv.fwd(self.A2, None, self.H2)
        E.gn_relu_fwd(tp, self.H2, g2["gamma"], g2["beta"], self.A3, g2["stats"], g2["G"])
        l2, li = self.lin2, self.lin_in
        terms = [dict(src=self.A3, op=-1, F=self.mid, src_rows=self.rows, src_stride=self.mid, w=l2.W3[:, 0, :],
                      w_stride=self.Fo, wT=l2.Wt[0], wT_stride=self.mid, wT_lo=l2.Wt_lo[0])]
        if li is not None:
            terms.append(dict(src=self.Z, op=-1, F=self.Ft, src_rows=self.rows, src_stride=self.Ft, w=li.W3[:, 0, :],
                              w_stride=self.Fo, wT=li.Wt[0], wT_stride=self.Ft, wT_lo=li.Wt_lo[0]))
        cheb_call(tp, N, self.rows, self.Fo, terms, out,
                  tag=("dec/res:out", l2.alg_bytes(N, "fwd") + (li.alg_bytes(N, "fwd") if li is not None else 0)))
        if li is None:
            axpy(tp, out, self.Z[:N], 1.0)               # identity skip connection

    def bwd(self, x, ycat, dout, dx, dycat):
        """dout: gradient w.r.t. the block output; dx: gradient w.r.t. the block input x (written); dycat +=."""
        tp, N = self.tp, dout.shape[0]
        g0, g1, g2 = self.gn
        self.lin2.bwd(self.A3, None, dout, dx=self.dA3)
        if self.lin_in is not None:
            self.lin_in.bwd(self.Z, None, dout, dx=self.dZ)
        else:
            self.dZ[:N].copy_(dout)
        E.gn_relu_bwd(tp, self.H2, self.A3, self.dA3, g2["gamma"], g2["stats"], self.dH2, g2["dgamma"], g2["dbeta"], g2["G"])
        self.conv.bwd(self.A2, None, self.dH2, dx=self.dA2)
        E.gn_relu_bwd(tp, self.H1, self.A2, self.dA2, g1["gamma"], g1["stats"], self.dH1, g1["dgamma"], g1["dbeta"], g1["G"])
        self.lin1.bwd(self.A1, None, self.dH1, dx=self.dA1)
        E.gn_relu_bwd(tp, self.Z, self.A1, self.dA1, g0["gamma"], g0["stats"], self.dZ, g0["dgamma"], g0["dbeta"], g0["G"],
                      accumulate_dx=True)
        # back through concat + unpool: feature channels with U^T, condition channels reduced over the vertices
        E.resample(tp, self.op_uT, self.dZ, dx, N, self.rows_in, self.rows, self.Fin, x_stride=self.Ft,
                   y_stride=dx.shape[2])
        colsum(tp, self.dZ[:, :, self.Fin:], N, self.rows, self.Cc, [self.op_u], dycat.view(N, 1, self.Cc),
               g_stride=self.Ft)


class EncResBlock:
    """Encoder residual block (res_block, lib/models.py:715-741) at level i:
        h1 = leaky(cheb_K(x; W1) + b1);   out = D leaky(cheb_K(h1; W2) + skip(x) + b2),
    skip = x when the channel counts match, else the 1x1 projection x Ws.  The pooling D selects rows, so it is folded
    into conv2's operators and into the skip.  conv2 and the skip are ONE launch: the projection is one more contracted
    term, the identity skip a pass-through term (cape_term without weights).  The first block's projection reads the
    3 coordinates (+ the condition channels), which would drop the fused launch to the fp32 kernel: it runs on the thin
    kernel into `xs` and enters the launch as a pass-through term.  The data gradient into x is one launch as well:
    sum_k T_k^T (dh1 W1_k^T) + D^T (g2 Ws^T) or + D^T g2."""

    def __init__(self, net, i, L, D, Fin, C, Fo, K, maxN, order_in=None, order_mid=None, order_out=None):
        w, g = net._w, net._g
        tp, dev = net.tp, net.device
        self.net, self.tp, self.i, self.C, self.Fin, self.Fo = net, tp, i, C, Fin, Fo
        sc = "generator/encoder/encoder_resblock%d/" % (i + 1)
        nm = "enc/res%d" % (i + 1)
        self.conv1 = ChebLayer(net, ConvSite(tp, L, K, order_in=order_in, order_out=order_mid), Fin, C, Fo,
                               w(sc + "filter_1/weights"), g(sc + "filter_1/weights"), bias=w(sc + "bias_relu_1/bias"),
                               gbias=g(sc + "bias_relu_1/bias"), act=ACT_LEAKY, need_dx=(i > 0), maxN=maxN,
                               name=nm + "/conv1", fused=True)
        self.conv2 = ChebLayer(net, ConvSite(tp, L, K, D=D, order_in=order_mid, order_out=order_out), Fo, 0, Fo,
                               w(sc + "filter_2/weights"), g(sc + "filter_2/weights"), bias=w(sc + "bias_relu_2/bias"),
                               gbias=g(sc + "bias_relu_2/bias"), act=ACT_LEAKY, maxN=maxN, name=nm + "/conv2", fused=True)
        self.skip = ConvSite(tp, L, 1, D=D, order_in=order_in, order_out=order_out)      # x -> D x
        self.proj = None
        if (sc + "1x1-conv/weights") in net.specs:
            self.proj = ChebLayer(net, self.skip, Fin, C, Fo, w(sc + "1x1-conv/weights"), g(sc + "1x1-conv/weights"),
                                  need_dx=False, maxN=maxN, name=nm + "/1x1")
        # thin projection (F <= 4 or condition channels): computed apart, added as a pass-through term
        self.xs = (torch.zeros(maxN, self.skip.rows_out, Fo, device=dev)
                   if self.proj is not None and (Fin % 4 != 0 or C > 0) else None)
        self.h1 = torch.zeros(maxN, self.conv1.site.rows_out, Fo, device=dev)
        self.dh1 = torch.zeros_like(self.h1)

    def layers(self):
        return [l for l in (self.conv1, self.conv2, self.proj) if l is not None]

    def fwd(self, x, ycat, out):
        N, sx, sk = x.shape[0], x.shape[2], self.skip
        h1 = self.h1[:N]
        self.conv1.fwd(x, ycat, h1)
        if self.xs is not None:
            self.proj.fwd(x, ycat, self.xs[:N])
            t = dict(src=self.xs[:N], op=-1, F=self.Fo, src_rows=sk.rows_out, src_stride=self.Fo, w=None, w_stride=0)
        elif self.proj is not None:
            p = self.proj
            t = dict(src=x, op=sk.ops[0], F=self.Fin, src_rows=sk.rows_in, src_stride=sx, w=p.W3[:, 0, :],
                     w_stride=self.Fo, wT=p.Wt[0], wT_stride=self.Fin, wT_lo=p.Wt_lo[0])
            if p.stash_a[0] is not None:
                t["stash"], t["stash_stride"] = p.stash_a[0][:N], self.Fin
        else:
            t = dict(src=x, op=sk.ops[0], F=self.Fin, src_rows=sk.rows_in, src_stride=sx, w=None, w_stride=0)
        self.conv2.fwd(h1, None, out, extra=[t])

    def bwd(self, x, ycat, g2, dx=None, dx_aux=None, dycat=None):
        """g2: gradient w.r.t. conv2's pre-activation (the block's output rows); dx (written, SLOPE epilogue with the
        producing block's output dx_aux) when the block has an input gradient; dycat +=."""
        N, sk = g2.shape[0], self.skip
        h1, dh1 = self.h1[:N], self.dh1[:N]
        self.conv2.bwd(h1, None, g2, dx=dh1, dx_epi=EPI_SLOPE, dx_aux=h1)
        if self.proj is not None:
            self.proj.bwd(x, ycat, g2, dycat=dycat)             # weight (and condition) gradients of the projection
        if dx is None:
            self.conv1.bwd(x, ycat, dh1, dycat=dycat)
            return
        if self.proj is not None:
            p = self.proj
            t = dict(src=g2, op=sk.opsT[0], F=self.Fo, src_rows=sk.rows_out, src_stride=self.Fo, w=p.Wt[0],
                     w_stride=self.Fin, wT=p.W3[:, 0, :], wT_stride=self.Fo, wT_lo=p.W3_lo[:, 0, :])
        else:
            t = dict(src=g2, op=sk.opsT[0], F=self.Fo, src_rows=sk.rows_out, src_stride=self.Fo, w=None, w_stride=0)
        self.conv1.bwd(x, ycat, dh1, dx=dx, dx_epi=EPI_SLOPE, dx_aux=dx_aux, dycat=dycat, dx_extra=[t])


class CapeNetwork:
    """Encoder/decoder/discriminator + losses + optimiser on one GPU for a fixed batch size."""

    def __init__(self, L, D, U, L_d, D_d, cfg, batch_size, device=0, params=None, ref_compat=False, reorder=None):
        """reorder: keep the hidden activations in patch order (topology.patch_order) instead of the reference's
        vertex numbering.  Everything visible from outside (inputs, outputs, parameters, their gradients, the
        FC-layer row layout) stays in the reference numbering: the permutations are folded into the operator
        tables of the first/last conv of each stack.  Default: off (env CAPE_REORDER=1 turns it on): a gather batch
        waits for its slowest load whatever the L1 hit rate; kept because the shared-memory halo staging planned next needs compact tiles."""
        self.cfg = dict(cfg)
        if reorder is None:
            reorder = os.environ.get("CAPE_REORDER", "0") == "1"
        self.reorder = bool(reorder)
        self.N = int(batch_size)
        self.ref_compat = bool(ref_compat)
        c = self.cfg
        if not c["use_res_block_dec"] or c["reduce_dim"] <= 0:
            raise NotImplementedError("the plain decoder (use_res_block_dec=0) and reduce_dim=0 are not built")
        if c["optimizer"] not in ("sgd", "adam") or c["loss"] != "l1":
            raise NotImplementedError("optimizer must be 'sgd' (momentum) or 'adam' (lib/models.py:449-453); only "
                                      "loss='l1' is implemented")
        self.adam = c["optimizer"] == "adam"
        self.adam_t = 0                     # optimiser applications so far (TF: beta1_power = beta1 ** (adam_t + 1))
        self.tp = tp = Topology(device)
        self.device = dev = tp.device
        torch.cuda.set_device(dev)
        # Weight gradients on plain tensors (stashes) depend on nothing but their layer's operands, so they run on a
        # second stream next to the data-gradient chain and fill the ramp-up / tail bubbles of its kernels.  They get
        # a handle of their own (no operators, its own split-K workspace).
        self.dp = None                      # set_data_parallel(): bucketed gradient all-reduce inside the step
        self.async_dw = os.environ.get("CAPE_ASYNC_DW", "1") != "0"
        self.tp_dw = Topology(device) if self.async_dw else tp
        self.dw_stream = torch.cuda.Stream(device=dev) if self.async_dw else None
        self._dw_pending = False
        # column sums (bias / condition-channel gradients) off the main stream, their small products in ONE launch at the
        # end of the backward pass (CAPE_SIDE_GLUE=0: in line, one launch per player)
        self.side_glue = self.async_dw and os.environ.get("CAPE_SIDE_GLUE", "1") != "0"
        self.p = [int(l.shape[0]) for l in L]
        self.p_d = [int(l.shape[0]) for l in L_d]
        F, K, Kd = c["F"], c["K"], c["Kd"]
        nz, Cc = c["nz"], c["nz_cond"] + c["nz_cond2"]
        self.nz, self.Cc = nz, Cc
        N = self.N
        self.specs = specs = param_specs(c, self.p, self.p_d)
        gnames = [n for n in specs if is_g_param(n, True)]          # condition nets live in the G store
        dnames = [n for n in specs if is_d_param(n)]
        self.PG, self.PD = ParamStore(specs, gnames, dev), ParamStore(specs, dnames, dev)
        if self.adam:
            self.PG.add_adam_slot()
            self.PD.add_adam_slot()
        vals = params if params is not None else init_params(specs, c["seed"])
        self.PG.load(vals)
        self.PD.load(vals)
        self.arena = Arena()
        self.wprep = E.WeightPrep(tp)
        self.small = E.SmallGemmBatch(tp)
        self._scratch_need = 4
        self.ones = torch.ones(1, 2 * N, device=dev)
        w, g = self._w, self._g

        # ---- sites -------------------------------------------------------------------------------------
        nl = len(F)
        if self.reorder:
            og = topo.level_orders(L[0], D[:nl])
            od = topo.level_orders(L_d[0], D_d)
        else:
            og, od = [None] * (nl + 1), [None] * (len(D_d) + 1)
        self.order_g, self.order_d = og, od
        self.enc = []
        self.enc_res = bool(c["use_res_block"])
        self.cond_enc = bool(c["cond_encoder"])        # the first encoder layer also sees [y | y2] (models.py:531-535)
        fin = c["nn_input_channel"]
        for i in range(nl):
            Ci = Cc if (self.cond_enc and i == 0) else 0
            oi = og[i] if i > 0 else None
            if self.enc_res:
                self.enc.append(EncResBlock(self, i, L[i], D[i], fin, Ci, F[i], K[i], N, order_in=oi, order_mid=og[i],
                                            order_out=og[i + 1]))
            else:
                site = ConvSite(tp, L[i], K[i], D=D[i], order_in=oi, order_out=og[i + 1])
                sc = "generator/encoder/encoder_conv%d" % (i + 1)
                self.enc.append(ChebLayer(self, site, fin, Ci, F[i], w(sc + "/weights"), g(sc + "/weights"),
                                          bias=w(sc + "/bias"), gbias=g(sc + "/bias"), act=ACT_LEAKY, need_dx=(i > 0),
                                          maxN=N, name="enc/conv%d" % (i + 1)))
            fin = F[i]
        red = specs["generator/encoder/1x1-conv/weights"][1]
        self.red = red
        self.enc_1x1 = ChebLayer(self, ConvSite(tp, L[-1], 1, order_in=og[nl]), F[-1], 0, red,
                                 w("generator/encoder/1x1-conv/weights"),
                                 g("generator/encoder/1x1-conv/weights"), maxN=N, name="enc/1x1")
        flat = self.p[-1] * red
        self.flat = flat
        dn = lambda s, act=ACT_NONE: Dense(self, w(s + "/dense/kernel").view(specs[s + "/dense/kernel"]),
                                           w(s + "/dense/bias"), g(s + "/dense/kernel").view(specs[s + "/dense/kernel"]),
                                           g(s + "/dense/bias"), act, name=s.split("/", 1)[-1])
        self.fc_mean, self.fc_var = dn("generator/encoder/fc_mean"), dn("generator/encoder/fc_var")
        self.dec_fc1 = dn("generator/decoder/fc1", ACT_LEAKY)
        self.dec_1x1 = ChebLayer(self, ConvSite(tp, L[-1], 1, order_out=og[nl]), red, 0, F[-1],
                                 w("generator/decoder/1x1-conv/weights"),
                                 g("generator/decoder/1x1-conv/weights"), maxN=N, name="dec/1x1")
        self.dec = []
        self.affine = bool(c["affine"])
        fin = F[-1]
        for i in range(nl):
            if self.affine:
                Fo = F[-i - 1] // 2
                site = ConvSite(tp, L[-i - 2], K[-i - 1], U=U[-i - 1], order_in=og[nl - i], order_out=og[nl - i - 1])
                sc = "generator/decoder/decoder_resblock_affine%d" % (i + 1)
                self.dec.append(ChebLayer(self, site, fin, Cc, Fo, w(sc + "/graph_conv/weights"),
                                          g(sc + "/graph_conv/weights"), Wa=w(sc + "/affine/weights"),
                                          gWa=g(sc + "/affine/weights"), maxN=N, name="dec/aff%d" % (i + 1)))
            else:
                Fo = F[-i - 1]
                self.dec.append(GNBlock(self, i, L[-i - 2], U[-i - 1], fin, Cc, Fo, K[-i - 1],
                                        "generator/decoder/decoder_resblock_cmr%d" % (i + 1), N,
                                        order_in=og[nl - i], order_out=og[nl - i - 1]))
            fin = Fo
        self.dec_out = ChebLayer(self, ConvSite(tp, L[0], K[0], order_in=og[0]), fin, Cc, c["nn_input_channel"],
                                 w("generator/decoder/outputs/weights"), g("generator/decoder/outputs/weights"),
                                 bias=w("generator/decoder/outputs/bias"), gbias=g("generator/decoder/outputs/bias"),
                                 bias_per_row=True, maxN=N, name="dec/outputs")
        self.disc = []
        fin = c["nn_input_channel"]
        for i in range(len(D_d)):
            site = ConvSite(tp, L_d[i], Kd, D=D_d[i], order_in=od[i] if i > 0 else None, order_out=od[i + 1])
            sc = "discriminator/shared/conv%d" % (i + 1)
            self.disc.append(ChebLayer(self, site, fin, Cc if i == 0 else 0, F[i], w(sc + "/weights"),
                                       g(sc + "/weights"), bias=w(sc + "/bias"), gbias=g(sc + "/bias"), act=ACT_LEAKY,
                                       maxN=2 * N, n_cs_slots=2, name="disc/conv%d" % (i + 1)))
            fin = F[i]
        self.disc_pred = ChebLayer(self, ConvSite(tp, L_d[-1], K[-1], order_in=od[-1], order_out=od[-1]), fin, 0, 1,
                                   w("discriminator/prediction_map/weights"), g("discriminator/prediction_map/weights"),
                                   maxN=2 * N, n_cs_slots=2, name="disc/pred_map")
        # condition nets (models.py:479-511)
        self.c_pose1 = dn("condition_pose/fc1", ACT_LEAKY)
        self.c_pose2 = dn("condition_pose/fc2")
        if "condition_clo_label/fc2/dense/kernel" in specs:
            self.c_clo1, self.c_clo2 = dn("condition_clo_label/fc1", ACT_LEAKY), dn("condition_clo_label/fc2")
        else:
            self.c_clo1, self.c_clo2 = dn("condition_clo_label/fc1"), None
        self.nbr_op = tp.add_operator(_adjacency(L[0]))
        self.n_edges = int(_adjacency(L[0]).nnz // 2)
        self.arena.build(dev)
        self.scratch = torch.empty(self._scratch_need, device=dev)

        # ---- buffers -----------------------------------------------------------------------------------
        z = lambda *s: torch.zeros(*s, device=dev)
        P0 = self.p[0]
        ci, c2i = c["cond_dim"], c["cond2_dim"]
        self.in_x = z(N, P0, 3)                 # generator input (also its reconstruction target)
        self.in_cond = z(2 * N, ci)             # rows [0,N): discriminator batch, [N,2N): generator batch
        self.in_cond2 = z(2 * N, c2i)
        self.in_eps = z(N, nz)
        self.xcat = z(2 * N, P0, 3)             # [x_real ; x_hat]
        self.x_hat = self.xcat[N:]
        self.ycat = z(2 * N, Cc)                # [y | y2] for both batches
        self.ycat_g = self.ycat[N:]
        h1 = specs["condition_pose/fc1/dense/kernel"][1]
        self.cp_h = z(2 * N, h1)
        self.cc_h = z(2 * N, specs["condition_clo_label/fc1/dense/kernel"][1]) if self.c_clo2 else None
        enc_shape = [(l.conv2.site.rows_out, l.Fo) if self.enc_res else (l.site.rows_out, l.Fout) for l in self.enc]
        self.enc_act = [z(N, *s) for s in enc_shape]
        self.enc_red = z(N, self.p[-1], red)
        self.z_mean, self.z_logvar = z(N, nz), z(N, nz)
        self.z_total = z(N, nz + Cc)
        self.dec_fc = z(N, flat)
        self.dec_h0 = z(N, self.p[-1], F[-1])
        if self.affine:
            self.dec_act = [z(N, l.site.rows_out, l.Fout) for l in self.dec]
            self.dec_rg = [z(N, l.site.rows_out, l.Fout) for l in self.dec]
        else:
            self.dec_act = [z(N, b.rows, b.Fo) for b in self.dec]
            self.dec_rg = []
        self.disc_act = [z(2 * N, l.site.rows_out, l.Fout) for l in self.disc]
        self.logits = z(2 * N, self.p_d[-1], 1)
        # gradients
        self.d_logits = z(2 * N, self.p_d[-1], 1)
        self.d_logits_g = z(N, self.p_d[-1], 1)
        self.g_disc = [z(2 * N, l.site.rows_out, l.Fout) for l in self.disc]
        self.d_xhat = z(N, P0, 3)
        self.d_ycat = z(N, Cc)
        self.g_dec = [torch.zeros_like(a) for a in self.dec_act]             # d out of each block
        self.g_dec_m = [torch.zeros_like(a) for a in self.dec_act] if self.affine else []   # masked (graph-conv branch)
        self.g_dec_h0 = z(N, self.p[-1], F[-1])
        self.g_dec_fc = z(N, flat)
        self.g_dec_fc_t = z(N, flat)
        self.g_z = z(N, nz)
        self.g_mean, self.g_logvar = z(N, nz), z(N, nz)
        self.g_enc_red = z(N, self.p[-1], red)
        self.g_enc = [z(N, *s) for s in enc_shape]
        self.g_cp_h, self.g_cp_t = z(N, h1), z(N, h1)
        self.g_cc_h = z(N, self.cc_h.shape[1]) if self.c_clo2 else None
        self.g_cc_t = z(N, self.cc_h.shape[1]) if self.c_clo2 else None
        self.losses = z(8)       # recon, edge, kl, gan_g, gan_d_real, gan_d_fake
        self.sumsq = z(2)
        self.lr = z(2)
        self._lr_host = torch.zeros(256, 2).pin_memory()   # ring: the async H2D of step k must not see step k+1's value
        self._lr_slot = 0
        self.step_count = 0
        # workspace: split-K partials (dW of the widest layer, FC split-K)
        tp.reserve_workspace(64 << 20)
        if self.async_dw:
            self.tp_dw.reserve_workspace(64 << 20)
        self.prep_weights()

    # ---- parameter access --------------------------------------------------------------------------------
    def _store(self, n):
        return self.PD if is_d_param(n) else self.PG

    def _w(self, n):
        return self._store(n).w(n)

    def _g(self, n):
        return self._store(n).g(n)

    def get_params(self):
        out = self.PG.export()
        out.update(self.PD.export())
        return out

    def get_grads(self):
        out = self.PG.export(self.PG.grad)
        out.update(self.PD.export(self.PD.grad))
        return out

    def set_params(self, vals):
        self.PG.load(vals)
        self.PD.load(vals)
        self.prep_weights()

    def all_layers(self):
        dec = self.dec if self.affine else [l for b in self.dec for l in b.layers()]
        enc = [l for b in self.enc for l in b.layers()] if self.enc_res else self.enc
        return enc + [self.enc_1x1, self.dec_1x1] + dec + [self.dec_out] + self.disc + [self.disc_pred]

    def run_dw(self, fn):
        """Issue the weight-gradient launches `fn(topology)` of one layer: on the side stream (after everything
        enqueued so far on the main one) or, when profiling per launch / CAPE_ASYNC_DW=0, in line."""
        if not self.async_dw or E.PROFILE is not None:
            fn(self.tp)
            return
        ev = torch.cuda.Event()
        ev.record()
        self.dw_stream.wait_event(ev)
        with torch.cuda.stream(self.dw_stream):
            fn(self.tp_dw)
        self._dw_pending = True

    def run_glue(self, fn):
        """Issue a launch whose result only the deferred small products read (bias / condition column sums): on the side
        stream behind the layer's weight gradients when `side_glue` is on, else in line on the main stream."""
        if self.side_glue:
            self.run_dw(lambda _tp: fn())
        else:
            fn()

    def join_dw(self):
        if self._dw_pending:
            torch.cuda.current_stream().wait_stream(self.dw_stream)
            self._dw_pending = False

    def lo_of(self, t):
        r = self.PG.lo_of(t)
        return r if r is not None else self.PD.lo_of(t)

    def prep_weights(self):
        """Copies derived from the weights (K-major / per-order layouts, tf32 low parts); run after every update:
        three launches for the whole network."""
        E.tf32_lo(self.tp, self.PG.flat, self.PG.lo)
        E.tf32_lo(self.tp, self.PD.flat, self.PD.lo)
        self.wprep.run()

    def scratch_req(self, nfloats):
        """Layers announce the size of the intermediate their split forms need (Z = X @ [W_k]: consumed by the next
        launch on the same stream, so one buffer serves every layer)."""
        self._scratch_need = max(getattr(self, "_scratch_need", 4), int(nfloats))

    # ---- inputs --------------------------------------------------------------------------------------------
    def set_inputs(self, x_g, cond_g, cond2_g, eps, x_d=None, cond_d=None, cond2_d=None, non_blocking=True):
        """Host (pinned) or device tensors -> device input buffers."""
        N = self.N
        self.in_x.copy_(x_g, non_blocking=non_blocking)
        self.in_cond[N:].copy_(cond_g, non_blocking=non_blocking)
        self.in_cond2[N:].copy_(cond2_g, non_blocking=non_blocking)
        self.in_eps.copy_(eps, non_blocking=non_blocking)
        if x_d is not None:
            self.xcat[:N].copy_(x_d, non_blocking=non_blocking)
            self.in_cond[:N].copy_(cond_d, non_blocking=non_blocking)
            self.in_cond2[:N].copy_(cond2_d, non_blocking=non_blocking)

    def prefetch_inputs(self, x_g, cond_g, cond2_g, eps, x_d=None, cond_d=None, cond2_d=None):
        """Start the host->device copy of the NEXT step's batch (pinned host tensors) on a side stream, into one of two
        staging sets; `commit_inputs()` makes it the current batch.  The copy overlaps the step that is running."""
        if not hasattr(self, "_stage"):
            bufs = (self.in_x, self.in_cond[self.N:], self.in_cond2[self.N:], self.in_eps, self.xcat[:self.N],
                    self.in_cond[:self.N], self.in_cond2[:self.N])
            self._stage = [[torch.empty_like(b) for b in bufs] for _ in range(2)]
            self._stage_ev = [torch.cuda.Event(), torch.cuda.Event()]
            self._stage_free = [torch.cuda.Event(), torch.cuda.Event()]
            self._copy_stream = torch.cuda.Stream(device=self.device)
            self._stage_slot = 0
            for e in self._stage_free:
                e.record()
        slot = self._stage_slot
        self._copy_stream.wait_event(self._stage_free[slot])        # its previous contents have been consumed
        srcs = (x_g, cond_g, cond2_g, eps) if x_d is None else (x_g, cond_g, cond2_g, eps, x_d, cond_d, cond2_d)
        self._stage_n = len(srcs)                 # generator-only batches (forward / inference) stage four tensors
        with torch.cuda.stream(self._copy_stream):
            for dst, src in zip(self._stage[slot], srcs):
                dst.copy_(src, non_blocking=True)
            self._stage_ev[slot].record(self._copy_stream)

    def commit_inputs(self):
        """Make the batch started by the last `prefetch_inputs` the current one (device-to-device, compute stream)."""
        slot = self._stage_slot
        cur = torch.cuda.current_stream()
        cur.wait_event(self._stage_ev[slot])
        self.set_inputs(*self._stage[slot][: self._stage_n])
        self._stage_free[slot].record(cur)
        self._stage_slot = 1 - slot

    # ---- forward pieces ---------------------------------------------------------------------------------------
    def cond_fwd(self, lo, hi):
        """condition nets on rows [lo,hi) of the stacked condition inputs -> ycat rows."""
        nzc = self.cfg["nz_cond"]
        self.c_pose1.fwd(self.in_cond[lo:hi], self.cp_h[lo:hi])
        self.c_pose2.fwd(self.cp_h[lo:hi], self.ycat[lo:hi, :nzc])
        if self.c_clo2 is None:
            self.c_clo1.fwd(self.in_cond2[lo:hi], self.ycat[lo:hi, nzc:])
        else:
            self.c_clo1.fwd(self.in_cond2[lo:hi], self.cc_h[lo:hi])
            self.c_clo2.fwd(self.cc_h[lo:hi], self.ycat[lo:hi, nzc:])

    def encoder_fwd(self):
        x = self.in_x
        yc = self.ycat_g if self.cond_enc else None       # the generator batch's condition embeddings
        for l, a in zip(self.enc, self.enc_act):
            l.fwd(x, yc, a)
            x, yc = a, None
        self.enc_1x1.fwd(x, None, self.enc_red)
        flat = self.enc_red.view(self.N, self.flat)
        self.fc_mean.fwd(flat, self.z_mean)
        self.fc_var.fwd(flat, self.z_logvar)

    def sample_fwd(self):
        N, nz = self.N, self.nz
        _lib.check(self.tp.lib.cape_vae_sample_fwd(E._ptr(self.z_mean), E._ptr(self.z_logvar), E._ptr(self.in_eps),
                                                   E._ptr(self.z_total), nz + self.Cc, N, nz, E._stream()))
        self.z_total[:, nz:].copy_(self.ycat_g)

    def decoder_fwd(self, z_total=None, ycat=None, out=None):
        z_total = self.z_total if z_total is None else z_total
        ycat = self.ycat_g if ycat is None else ycat
        out = self.x_hat if out is None else out
        self.dec_fc1.fwd(z_total, self.dec_fc)
        self.dec_1x1.fwd(self.dec_fc.view(self.N, self.p[-1], self.red), None, self.dec_h0)
        x = self.dec_h0
        if self.affine:
            for l, a, rg in zip(self.dec, self.dec_act, self.dec_rg):
                l.fwd(x, ycat, a, out2=rg)
                x = a
        else:
            for b, a in zip(self.dec, self.dec_act):
                b.fwd(x, ycat, a)
                x = a
        self.dec_out.fwd(x, ycat, out)

    def disc_fwd(self, lo, hi):
        x = self.xcat[lo:hi]
        yc = self.ycat[lo:hi]
        for l, a in zip(self.disc, self.disc_act):
            l.fwd(x, yc, a[lo:hi])
            x = a[lo:hi]
        self.disc_pred.fwd(x, None, self.logits[lo:hi])

    # ---- backward pieces ---------------------------------------------------------------------------------------
    def disc_bwd(self, lo, hi, dlogits, want_dw, dx=None, dycat=None, cs_slot=0):
        """dlogits: [hi-lo, 431, 1] upstream gradient.  want_dw: discriminator-loss path (weight grads);
        dx/dycat: generator-loss path (gradient w.r.t. the input mesh and the condition embedding)."""
        n = len(self.disc)
        acts = [a[lo:hi] for a in self.disc_act]
        gs = [gb[: hi - lo] for gb in self.g_disc]
        yc = self.ycat[lo:hi]
        self.disc_pred.bwd(acts[-1], None, dlogits, dx=gs[-1], dx_epi=EPI_SLOPE, dx_aux=acts[-1], want_dw=want_dw,
                           cs_slot=cs_slot)
        for i in range(n - 1, 0, -1):
            self.disc[i].bwd(acts[i - 1], None, gs[i], dx=gs[i - 1], dx_epi=EPI_SLOPE, dx_aux=acts[i - 1],
                             want_dw=want_dw, cs_slot=cs_slot)
        self.disc[0].bwd(self.xcat[lo:hi], yc, gs[0], dx=dx, dycat=dycat, want_dw=want_dw, cs_slot=cs_slot)

    def decoder_bwd(self):
        """d_xhat -> decoder weight grads, d z_total, d ycat (accumulated)."""
        N, nl = self.N, len(self.dec)
        yc = self.ycat_g
        last = self.dec_act[-1]
        if not self.affine:
            self.dec_out.bwd(last, yc, self.d_xhat, dx=self.g_dec[-1], dycat=self.d_ycat)
            for i in range(nl - 1, -1, -1):
                x = self.dec_act[i - 1] if i > 0 else self.dec_h0
                self.dec[i].bwd(x, yc, self.g_dec[i], self.g_dec[i - 1] if i > 0 else self.g_dec_h0, self.d_ycat)
        else:
            self.dec_out.bwd(last, yc, self.d_xhat, dx=self.g_dec[-1], dx2=self.g_dec_m[-1], dx_epi=EPI_DUALMASK,
                             dx_aux=self.dec_rg[-1], dycat=self.d_ycat)
        for i in range(nl - 1 if self.affine else -1, -1, -1):
            x = self.dec_act[i - 1] if i > 0 else self.dec_h0
            if i > 0:
                self.dec[i].bwd(x, yc, self.g_dec_m[i], g_aff=self.g_dec[i], dx=self.g_dec[i - 1],
                                dx2=self.g_dec_m[i - 1], dx_epi=EPI_DUALMASK, dx_aux=self.dec_rg[i - 1],
                                dycat=self.d_ycat)
            else:
                self.dec[i].bwd(x, yc, self.g_dec_m[i], g_aff=self.g_dec[i], dx=self.g_dec_h0, dycat=self.d_ycat)
        fcv = self.dec_fc.view(N, self.p[-1], self.red)
        self.dec_1x1.bwd(fcv, None, self.g_dec_h0, dx=self.g_dec_fc.view(N, self.p[-1], self.red))
        self.dec_fc1.bwd(self.z_total, self.dec_fc, self.g_dec_fc, gtmp=self.g_dec_fc_t)
        W = self.dec_fc1.W                     # [nz + Cc, flat]: rows [0,nz) latent code, rows [nz,..) condition (models.py:641)
        gemm(self.tp, self.g_dec_fc_t, W[:self.nz].t(), self.g_z)
        gemm(self.tp, self.g_dec_fc_t, W[self.nz:].t(), self.d_ycat, beta=1.0)

    def encoder_bwd(self):
        N, nz = self.N, self.nz
        c = self.cfg
        _lib.check(self.tp.lib.cape_vae_sample_bwd(E._ptr(self.g_z), nz, E._ptr(self.z_mean),
                                                   E._ptr(self.z_logvar), E._ptr(self.in_eps), E._ptr(self.g_mean),
                                                   E._ptr(self.g_logvar), N, nz, float(c["lambda_latent"]),
                                                   E._stream()))
        flat = self.enc_red.view(N, self.flat)
        gflat = self.g_enc_red.view(N, self.flat)
        self.fc_mean.bwd(flat, self.z_mean, self.g_mean, dx=gflat)
        self.fc_var.bwd(flat, self.z_logvar, self.g_logvar, dx=gflat, dx_beta=1.0)
        self._fc_reg(("generator/encoder/fc_mean", "generator/encoder/fc_var"))
        self._reduce_bucket("enc_fc")                       # 28 MB of gradients are final: all-reduce behind the conv backward
        self.enc_1x1.bwd(self.enc_act[-1], None, self.g_enc_red, dx=self.g_enc[-1], dx_epi=EPI_SLOPE,
                         dx_aux=self.enc_act[-1])
        yc = self.ycat_g if self.cond_enc else None
        dyc = self.d_ycat if self.cond_enc else None        # complete before cond_bwd (the small products flush first)
        for i in range(len(self.enc) - 1, 0, -1):
            if self.enc_res:
                self.enc[i].bwd(self.enc_act[i - 1], None, self.g_enc[i], dx=self.g_enc[i - 1],
                                dx_aux=self.enc_act[i - 1])
            else:
                self.enc[i].bwd(self.enc_act[i - 1], None, self.g_enc[i], dx=self.g_enc[i - 1], dx_epi=EPI_SLOPE,
                                dx_aux=self.enc_act[i - 1])
        self.enc[0].bwd(self.in_x, yc, self.g_enc[0], dycat=dyc)

    def cond_bwd(self):
        """d_ycat (generator batch) -> condition-net weight grads."""
        N = self.N
        nzc = self.cfg["nz_cond"]
        dy = self.d_ycat[:, :nzc]
        dy2 = self.d_ycat[:, nzc:]
        self.c_pose2.bwd(self.cp_h[N:], None, dy, dx=self.g_cp_h)
        self.c_pose1.bwd(self.in_cond[N:], self.cp_h[N:], self.g_cp_h, gtmp=self.g_cp_t)
        if self.c_clo2 is None:
            self.c_clo1.bwd(self.in_cond2[N:], None, dy2)
        else:
            self.c_clo2.bwd(self.cc_h[N:], None, dy2, dx=self.g_cc_h)
            self.c_clo1.bwd(self.in_cond2[N:], self.cc_h[N:], self.g_cc_h, gtmp=self.g_cc_t)

    # ---- public passes ------------------------------------------------------------------------------------------
    def forward_generator(self):
        """condition nets + encoder + sampling + decoder on the generator batch (BASELINE config 2)."""
        N = self.N
        self.cond_fwd(N, 2 * N)
        self.encoder_fwd()
        self.sample_fwd()
        self.decoder_fwd()
        return self.x_hat

    def lr_now(self, step):
        """Learning-rate policy of CAPE.training (lib/models.py:426-442)."""
        c = self.cfg
        lr_g, lr_d = c["lr"], c["lr"] * c["lr_scaler"]
        ds = int(c["decay_steps"])
        if c["lr_warmup"]:
            warm = int(c["decay_steps"] * 8)
            if step < warm:
                return lr_g * step / warm, lr_d * step / warm
            k = math.floor((step - warm) / ds)
        else:
            k = math.floor(step / ds)
        return lr_g * c["decay_rate"] ** k, lr_d * c["decay_rate"] ** k

    def enqueue_fwd_bwd(self):
        """Forward + backward of both players for the staged batch; pure device work (CUDA-graph capturable)."""
        N, c, tp = self.N, self.cfg, self.tp
        lam_gan = float(c["lambda_gan"])
        self.arena.zero()
        self.losses.zero_()
        self.d_ycat.zero_()
        if not self.affine:
            self.PG.grad.zero_()          # group-norm gamma/beta gradients are accumulated by their kernels
        # forward: both condition batches at once, generator, discriminator on [real ; fake]
        self.cond_fwd(0, 2 * N)
        self.encoder_fwd()
        self.sample_fwd()
        self.decoder_fwd()
        self.disc_fwd(0, 2 * N)
        nlog = N * self.p_d[-1]
        L = self.losses
        lib = tp.lib
        st = E._stream
        # GAN losses with soft labels 0.9 / 0.1 (models.py:383-390)
        _lib.check(lib.cape_bce_logits(E._ptr(self.logits[N:]), nlog, 0.9, lam_gan, E._ptr(self.d_logits_g),
                                       E._ptr(L[3:]), st()))
        _lib.check(lib.cape_bce_logits(E._ptr(self.logits[:N]), nlog, 0.9, lam_gan, E._ptr(self.d_logits[:N]),
                                       E._ptr(L[4:]), st()))
        _lib.check(lib.cape_bce_logits(E._ptr(self.logits[N:]), nlog, 0.1, lam_gan, E._ptr(self.d_logits[N:]),
                                       E._ptr(L[5:]), st()))
        # discriminator-loss path: weight gradients from both halves
        if not self.ref_compat:
            self.disc_bwd(0, 2 * N, self.d_logits, want_dw=True)
        # generator-loss path through D(fake): gradient w.r.t. x_hat and the condition embedding (it rewrites the
        # gradient buffers the discriminator's weight gradients are still reading on the side stream: join first)
        self.join_dw()
        self.disc_bwd(N, 2 * N, self.d_logits_g, want_dw=False, dx=self.d_xhat, dycat=self.d_ycat, cs_slot=1)
        _lib.check(lib.cape_recon_losses(tp.h, self.nbr_op, E._ptr(self.x_hat), E._ptr(self.in_x), N, self.p[0],
                                         float(c["lambda_recon"]), float(c["lambda_edge"]), self.n_edges,
                                         E._ptr(self.z_mean), E._ptr(self.z_logvar), self.nz, E._ptr(self.d_xhat),
                                         E._ptr(L), st()))
        self.decoder_bwd()
        self._fc_reg(("generator/decoder/fc1",))
        if not self.side_glue:
            self.small.flush()        # bias / condition-channel gradients of the decoder and discriminator layers
        self._reduce_bucket("dec")    # decoder (+ discriminator) gradients are final: all-reduce behind the encoder backward
        self.encoder_bwd()
        # side_glue: the column sums ran on the side stream, so every small product of the step goes out in one launch
        # once that stream has joined (d_ycat, which the condition nets' backward reads, is complete after it)
        self.join_dw()
        self.small.flush()            # (not side_glue: the encoder's bias gradients)
        self.cond_bwd()
        if self.ref_compat:
            self.PD.grad.copy_(self.PD.flat)          # models.py:466: the D "gradients" are its variables
        if not c["optim_condnet"]:                    # models.py:455-458: condition nets excluded from vars_g
            for n in self.PG.names:
                if not n.startswith("generator"):
                    self.PG.g(n).zero_()
        self._reduce_bucket("rest")
        if self.dp is not None:
            torch.cuda.current_stream().wait_stream(self.dp["stream"])

    def _fc_reg(self, names):
        """fc L2 regularisation: regularization * sum(l2_regularizer(regularization)(W)) -> grad reg^2 * W (models.py:378)"""
        r2 = float(self.cfg["regularization"]) ** 2
        if r2 > 0:
            for n in names:
                axpy(self.tp, self._g(n + "/dense/kernel"), self._w(n + "/dense/kernel"), r2)

    # ---- data parallelism: bucketed gradient all-reduce overlapped with the backward pass -------------------------
    def set_data_parallel(self, world):
        """Opt-in (the default data-parallel step all-reduces the two flat gradient buffers between the two graphs:
        `train_step(allreduce=...)`).  One process per GPU, batch sharded (SURVEY.md 8e).  The flat generator gradient
        buffer is all-reduced in three buckets as soon as each is final -- decoder (+ the discriminator's buffer) after
        the decoder backward, the two 28 MB encoder FC kernels right after their weight gradients, the encoder convs /
        condition nets at the end -- on a communication stream that the backward pass does not wait for until its very
        end.  Checked eagerly on two GPUs (replicas bit-identical, gradients of the global batch); captured inside the
        forward/backward graph the step also completes, but destroying the process group afterwards hung in the one
        run the budget allowed, so `bench.py` and `CAPE.fit` keep the default.  world <= 1 switches it off."""
        if world <= 1:
            self.dp = None
            return
        self.side_glue = False            # the "dec" bucket needs the decoder's bias / condition gradients at its boundary
        P = self.PG
        names = P.names
        fc0 = P.offsets["generator/encoder/fc_mean/dense/kernel"]
        dec0 = P.offsets[next(n for n in names if n.startswith("generator/decoder"))]
        assert fc0 < dec0 and all(P.offsets[n] >= dec0 for n in names if n.startswith("generator/decoder"))
        self.dp = dict(world=world, stream=torch.cuda.Stream(device=self.device),
                       buckets={"dec": [P.grad[dec0:]] + ([] if self.ref_compat else [self.PD.grad]),
                                "enc_fc": [P.grad[fc0:dec0]], "rest": [P.grad[:fc0]]})

    def _reduce_bucket(self, which):
        if self.dp is None:
            return
        import torch.distributed as dist
        comm = self.dp["stream"]
        comm.wait_stream(torch.cuda.current_stream())
        if self._dw_pending:
            comm.wait_stream(self.dw_stream)          # weight gradients of the bucket still running on the side stream
        with torch.cuda.stream(comm):
            for b in self.dp["buckets"][which]:
                dist.all_reduce(b, op=dist.ReduceOp.AVG)

    def enqueue_update(self):
        """clip_by_global_norm(5.0) + MomentumOptimizer for both players (models.py:460-467) + weight re-layouts.
        Learning rates are read from device memory (set_lr), so this too is CUDA-graph capturable."""
        lib = self.tp.lib
        self.sumsq.zero_()
        for P, i in ((self.PG, 0), (self.PD, 1)):
            _lib.check(lib.cape_sumsq(E._ptr(P.grad), P.size, E._ptr(self.sumsq[i:]), E._stream()))
            if self.adam:
                _lib.check(lib.cape_adam_clip_update(E._ptr(P.flat), E._ptr(P.grad), E._ptr(P.mom), E._ptr(P.var), P.size,
                                                     E._ptr(self.sumsq[i:]), 5.0, E._ptr(self.lr[i:]), ADAM_BETA1,
                                                     ADAM_BETA2, ADAM_EPS, E._stream()))
            else:
                _lib.check(lib.cape_sgd_clip_update(E._ptr(P.flat), E._ptr(P.grad), E._ptr(P.mom), P.size,
                                                    E._ptr(self.sumsq[i:]), 5.0, E._ptr(self.lr[i:]),
                                                    float(self.cfg["momentum"]), E._stream()))
        self.prep_weights()

    def set_lr(self, step):
        lr_g, lr_d = self.lr_now(step)
        if self.adam:
            # AdamOptimizer folds its bias correction into the step size: lr_t = lr sqrt(1 - b2^t) / (1 - b1^t), t counting
            # the applications of this optimiser (both players are applied once per update, so they share t)
            t = self.adam_t + 1
            corr = math.sqrt(1.0 - ADAM_BETA2 ** t) / (1.0 - ADAM_BETA1 ** t)
            lr_g, lr_d = lr_g * corr, lr_d * corr
        slot = self._lr_host[self._lr_slot]
        self._lr_slot = (self._lr_slot + 1) % self._lr_host.shape[0]
        slot[0], slot[1] = lr_g, lr_d
        self.lr.copy_(slot, non_blocking=True)

    @staticmethod
    @contextlib.contextmanager
    def _no_collector():
        """Stream capture with Python's cyclic garbage collector held off.  A dead network it finds mid-capture would
        destroy its topology handles, and the cudaFree of that invalidates the capture; so dead cycles are collected
        first, while that is still safe."""
        gc.collect()
        was_enabled = gc.isenabled()
        gc.disable()
        try:
            yield
        finally:
            if was_enabled:
                gc.enable()

    def capture_graphs(self):
        """Capture forward/backward and the update into two CUDA graphs (the gradient all-reduce runs between
        them).  One eager step must have run before (lazy initialisations, workspace growth)."""
        self.graph_fb, self.graph_up = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
        torch.cuda.synchronize()
        with self._no_collector():
            with torch.cuda.graph(self.graph_fb):
                self.enqueue_fwd_bwd()
            with torch.cuda.graph(self.graph_up):
                self.enqueue_update()
        torch.cuda.synchronize()

    def capture_forward_graph(self):
        """Capture the generator forward (condition nets + encoder + sampling + decoder, BASELINE configs[1]) into one
        CUDA graph: `graph_fwd.replay()` then maps the staged inputs to `x_hat`."""
        self.graph_fwd = torch.cuda.CUDAGraph()
        torch.cuda.synchronize()
        with self._no_collector():
            with torch.cuda.graph(self.graph_fwd):
                self.forward_generator()
        torch.cuda.synchronize()

    def train_step(self, step=None, update=True, allreduce=None, use_graph=False):
        """One optimiser application on both players = one sess.run(op_train_*) of the reference
        (lib/models.py:460-472).  Inputs must have been staged with set_inputs()."""
        step = self.step_count if step is None else step
        if update:
            self.set_lr(step)
        if use_graph:
            self.graph_fb.replay()
        else:
            self.enqueue_fwd_bwd()
        if allreduce is not None and self.dp is None:
            allreduce(self.PG.grad, self.PD.grad)
        if update:
            if use_graph:
                self.graph_up.replay()
            else:
                self.enqueue_update()
            self.step_count = step + 1
            self.adam_t += 1
        return self.losses

    def loss_dict(self):
        """Host copy of the last step's loss terms (synchronises)."""
        v = self.losses.detach().cpu().numpy()
        c = self.cfg
        out = dict(recon=float(v[0]), edge=float(v[1]), latent=float(v[2]), gan_g=float(v[3]),
                   gan_d=float(v[4] + v[5]))
        out["loss_g_noreg"] = (out["gan_g"] * c["lambda_gan"] + out["recon"] * c["lambda_recon"]
                               + out["edge"] * c["lambda_edge"] + out["latent"] * c["lambda_latent"])
        out["loss_d"] = out["gan_d"] * c["lambda_gan"]
        return out


def _adjacency(L):
    import scipy.sparse as sp
    A = sp.csr_matrix(L, copy=True)
    A.setdiag(0)
    A.eliminate_zeros()
    A.data[:] = 1.0
    return A
