"""CPU oracle of the reference's default encoder -- TEST INFRASTRUCTURE ONLY.

`ResOracle` extends oracle.cape_oracle.Oracle with what the reference's default configuration
(configs/default_config.yaml: use_res_block 1, cond_encoder 1) adds to the encoder: the residual blocks of
lib/models.py:715-741 and the condition concat of :531-535, restated line by line.  Every other method, and
`train_update`, are the base oracle's, so the configurations it already covers behave exactly as before.
Branch-mask sites of a residual block are "enc%d_1" (bias_relu_1) and "enc%d_2" (bias_relu_2).
"""
import torch

from oracle import cape_oracle as O


class ResOracle(O.Oracle):
    def res_block(self, x_in, i, P, scope):
        """models.py:715-741 (encoder residual block at level i)."""
        x = self.chebyshev5(x_in, self.Lt[i], P[scope + "/filter_1/weights"], self.K[i])        # filter_1
        x = self.b1leakyrelu(x, P[scope + "/bias_relu_1/bias"], site="enc%d_1" % (i + 1))       # bias_relu_1
        x = self.chebyshev5(x, self.Lt[i], P[scope + "/filter_2/weights"], self.K[i])           # filter_2
        if x_in.shape[-1] != x.shape[-1]:                                                       # 1x1-conv
            x_in = self.chebyshev5(x_in, self.Lt[i], P[scope + "/1x1-conv/weights"], 1)
        x = x + x_in                                                                            # addition
        x = self.b1leakyrelu(x, P[scope + "/bias_relu_2/bias"], site="enc%d_2" % (i + 1))       # bias_relu_2
        return self.poolwT(x, self.Dm[i])                                                       # pooling

    def encoder(self, x, P, y=None, y2=None):
        """models.py:514-561; y / y2: the generator batch's condition embeddings (used with cond_encoder)."""
        if not self.cfg.get("use_res_block") and not self.cfg.get("cond_encoder"):
            return super().encoder(x, P)
        s = "generator/encoder/"
        if self.cfg.get("cond_encoder"):                                                        # :531-535
            x = torch.cat([x, self.fit_cond_dim(x, y), self.fit_cond_dim(x, y2)], -1)
        for i in range(len(self.F)):
            if self.cfg.get("use_res_block"):
                x = self.res_block(x, i, P, s + "encoder_resblock%d" % (i + 1))
            else:
                sc = s + "encoder_conv%d" % (i + 1)
                x = self.chebyshev5(x, self.Lt[i], P[sc + "/weights"], self.K[i])
                x = self.b1leakyrelu(x, P[sc + "/bias"], site="enc%d" % (i + 1))
                x = self.poolwT(x, self.Dm[i])
            self._keep("enc_act%d" % (i + 1), x)
        if self.reduce_dim > 0:
            x = self._keep("enc_red", self.chebyshev5(x, self.Lt[-1], P[s + "1x1-conv/weights"], 1))
        x = x.reshape(x.shape[0], -1)
        return self.dense(x, P, s + "fc_mean"), self.dense(x, P, s + "fc_var")

    def generator(self, x, y, y2, eps, P):
        """models.py:620-645 with the encoder seeing the condition embeddings."""
        z_mean, z_logvar = self.encoder(x, P, y, y2)
        z = z_mean + torch.sqrt(torch.exp(z_logvar)) * eps
        z_total = self._keep("z_total", torch.cat([z, y, y2], 1))
        return self.decoder_cond_vert(z_total, y, y2, P), z_mean, z_logvar


# ---------------------------------------------------------------------------------------------------------------------
# GPU-side helpers of the residual-encoder tests (CapeNetwork vs ResOracle)
# ---------------------------------------------------------------------------------------------------------------------
def cuda_masks(net, h, N):
    """parity.cuda_masks for a network whose encoder may be built of residual blocks: the branch decisions of every
    (leaky-)ReLU of the CUDA forward, in the reference's vertex numbering, keyed like ResOracle's sites."""
    import numpy as np
    import scipy.sparse as sp
    from cape_b200 import topology as T2
    masks, rows = {}, {}

    def sel(D):
        return None if T2.is_identity(D, tol=0) else torch.from_numpy(sp.csr_matrix(D).indices.astype(np.int64))

    def pos(a, order):
        m = (a > 0).cpu()
        return m if order is None else m[:, torch.from_numpy(T2.inverse_order(order))]

    for i, a in enumerate(net.enc_act):
        b = net.enc[i]
        key = "enc%d_2" % (i + 1) if net.enc_res else "enc%d" % (i + 1)
        masks[key] = pos(a, b.conv2.site.order_out if net.enc_res else b.site.order_out)
        r = sel(h["D"][i])
        if r is not None:
            rows[key] = r
        if net.enc_res:
            masks["enc%d_1" % (i + 1)] = pos(b.h1[:N], b.conv1.site.order_out)
    for i, a in enumerate(net.dec_rg):
        masks["dec%d" % (i + 1)] = pos(a, net.dec[i].site.order_out)
    if not net.affine:
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
    masks["l1_sign"] = torch.sign(net.x_hat - net.in_x).cpu()
    return masks, rows


def train_step(h, cfg, N=2, step=100, seed=123, fc_scale=0.05, reorder=None, use_graph=False):
    """One full VAE+GAN update of CapeNetwork against ResOracle's autograd, as parity.train_step does it: x_hat and the
    losses unmasked and with the CUDA branch decisions imposed, every gradient, clipped update and post-update parameter
    with them imposed.  Returns {name: relative error}."""
    import numpy as np
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
        o = ResOracle(h["L"], h["D"], h["U"], h["L_d"], h["D_d"], cfg)
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
