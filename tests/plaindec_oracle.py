"""CPU oracle of the reference's plain decoder (`--use_res_block_dec 0`) -- TEST INFRASTRUCTURE ONLY.

`PlainDecOracle` extends tests/options_oracle.OptOracle (and through it the residual-encoder oracle and
oracle.cape_oracle.Oracle) with the decoder lib/models.py builds when use_res_block_dec is off: after fc1 (and the 1x1
conv when reduce_dim > 0) and the condition concat, every layer is `udn` (models.py:173-191, called at :603) -- unpool,
Chebyshev filter on the finer level's Laplacian, then the model's brelu, which follows cfg["activation"] (tanh
included).  The branch-mask site of decoder layer i is "dec_conv<i>".  `reduce_dim 0` needs nothing new: the base
oracles already skip both 1x1 convs then (models.py:549-552,585-589).  With use_res_block_dec on it is OptOracle,
operation for operation.
"""
import numpy as np
import torch

import options_oracle as OO
import resblock_oracle as R
from oracle import cape_oracle as O


class PlainDecOracle(OO.OptOracle):
    def udn_layer(self, x, i, P, scope):
        """models.py:173-191: unpool -> filter (Laplacian of the finer level) -> brelu."""
        x = self.poolwT(x, self.Um[-i - 1])
        x = self.chebyshev5(x, self.Lt[-i - 2], P[scope + "/weights"], self.K[-i - 1])
        return self.b1leakyrelu(x, P[scope + "/bias"], site="dec_conv%d" % (i + 1))

    def decoder_cond_vert(self, z_total, y, y2, P):
        """models.py:564-617."""
        if self.cfg["use_res_block_dec"]:
            return super().decoder_cond_vert(z_total, y, y2, P)
        s = "generator/decoder/"
        x = self._keep("dec_fc", self.dense(z_total, P, s + "fc1", act="leaky", site="dec_fc1"))   # :582
        x = x.reshape(x.shape[0], self.p[-1], -1)                                # :584
        if self.reduce_dim > 0:
            x = self.chebyshev5(x, self.Lt[-1], P[s + "1x1-conv/weights"], 1)     # :588
        x = torch.cat([x, self.fit_cond_dim(x, y), self.fit_cond_dim(x, y2)], -1)  # :591-594
        for i in range(len(self.F)):
            x = self._keep("dec_act%d" % (i + 1), self.udn_layer(x, i, P, s + "decoder_conv%d" % (i + 1)))   # :603
            x = torch.cat([x, self.fit_cond_dim(x, y), self.fit_cond_dim(x, y2)], -1)  # :606-609
        x = self.chebyshev5(x, self.Lt[0], P[s + "outputs/weights"], self.K[0])   # :612
        return x + P[s + "outputs/bias"]                                          # :615-616


# ---------------------------------------------------------------------------------------------------------------------
# GPU-side helpers (CapeNetwork vs PlainDecOracle)
# ---------------------------------------------------------------------------------------------------------------------
def cuda_masks(net, h, N):
    """The branch decisions of every (leaky-)ReLU of the CUDA forward, in the reference's vertex numbering, keyed like
    PlainDecOracle's sites: resblock_oracle.cuda_masks, plus the plain decoder's layers."""
    if not net.plain_dec:
        return R.cuda_masks(net, h, N)
    masks, rows = R.cuda_masks(_AffineView(net), h, N)
    for i, (l, a) in enumerate(zip(net.dec, net.dec_act)):
        m = (a > 0).cpu()
        if l.site.order_out is not None:
            from cape_b200 import topology as T
            m = m[:, torch.from_numpy(T.inverse_order(l.site.order_out))]
        masks["dec_conv%d" % (i + 1)] = m
    return masks, rows


class _AffineView:
    """A plain-decoder network seen by resblock_oracle.cuda_masks: its decoder contributes no masks there."""

    def __init__(self, net):
        self._net = net
        self.affine, self.dec_rg = True, []

    def __getattr__(self, k):
        return getattr(self._net, k)


def train_step(h, cfg, N=2, step=100, seed=123, fc_scale=0.05, reorder=None, use_graph=False):
    """One full VAE+GAN update of CapeNetwork against PlainDecOracle's autograd, as resblock_oracle.train_step does it:
    x_hat and the losses unmasked and with the CUDA branch decisions imposed, every gradient, clipped update and
    post-update parameter with them imposed.  Returns {name: relative error}."""
    import parity
    from cape_b200 import topology as T
    from cape_b200.network import CapeNetwork
    from cape_b200.params import param_specs
    from cape_b200.synthetic import make_batch
    specs = param_specs(cfg, [l.shape[0] for l in h["L"]], [l.shape[0] for l in h["L_d"]])
    params = parity.calibrated_params(specs, seed, fc_scale)
    net = CapeNetwork(h["L"], h["D"], h["U"], h["L_d"], h["D_d"], cfg, N, params=params, reorder=reorder)
    tb = {k: torch.from_numpy(v) for k, v in make_batch(N, cfg["nz"], seed=seed).items()}
    net.set_inputs(tb["x_g"], tb["cond_g"], tb["cond2_g"], tb["eps"], tb["x_d"], tb["cond_d"], tb["cond2_d"])
    if use_graph:
        net.train_step(step=step, update=False)
        torch.cuda.synchronize()
        net.capture_graphs()
    net.train_step(step=step, use_graph=use_graph)
    torch.cuda.synchronize()
    got_loss, got_x = net.loss_dict(), net.x_hat.cpu().numpy()
    got_g, got_p = net.get_grads(), net.get_params()
    got_m = net.PG.export(net.PG.mom)
    got_m.update(net.PD.export(net.PD.mom))
    masks, rows = cuda_masks(net, h, N)
    out = {}
    for imposed in (False, True):
        o = PlainDecOracle(h["L"], h["D"], h["U"], h["L_d"], h["D_d"], cfg)
        if imposed:
            o.masks, o.mask_rows = masks, rows
        P = {k: torch.from_numpy(np.asarray(v, np.float32)) for k, v in params.items()}
        M = {k: torch.zeros_like(v) for k, v in P.items()}
        res = O.train_update(o, P, M, tb, step, T.smpl_edges())
        pre = "" if imposed else "unmasked "
        out[pre + "x_hat (vertex-L2)"] = parity.vertex_l2(got_x, res["x_hat"].numpy())
        out[pre + "x_hat (max-rel)"] = parity.rel(got_x, res["x_hat"].numpy())
        for k in ("recon", "edge", "latent", "gan_g", "gan_d"):
            out[pre + "loss " + k] = abs(got_loss[k] - res[k]) / max(abs(res[k]), 1e-30)
        if not imposed:
            continue
        for k, g in res["grads"].items():
            out["grad " + k] = parity.rel(got_g[k].reshape(-1), g.numpy().reshape(-1))
        for k, m in res["mom"].items():
            out["clipped-update " + k] = parity.rel(got_m[k].reshape(-1), m.numpy().reshape(-1))
        for k, v in P.items():
            out["param " + k] = parity.rel(got_p[k].reshape(-1), v.numpy().reshape(-1))
    return out
