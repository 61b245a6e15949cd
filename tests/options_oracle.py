"""CPU oracle of the reference's `--activation` and `--loss` switches -- TEST INFRASTRUCTURE ONLY.

`OptOracle` extends tests/resblock_oracle.ResOracle (and through it oracle.cape_oracle.Oracle) with the two choices
lib/models.py makes by name:

  * `self.brelu = getattr(self, activation)` (models.py:60): the bias + activation after every plain encoder layer
    (cnp, :166), both activations of a residual encoder block (:721,:734) and every discriminator layer (cnp_d, :805).
    Those are exactly the sites where the base oracles call `b1leakyrelu`, so that one method dispatches on
    cfg["activation"] here.  b1relu honours imposed branch masks like the leaky sites; b1tanh has no branches.  The fixed
    activations (condition nets, decoder fc1, GroupNorm and affine decoder blocks) do not go through it and stay as
    they are.
  * the reconstruction loss of `loss()` (:357-369): 'l1' absolute_difference, 'huber' huber_loss(delta=0.1), any other
    string mean_squared_error, all Reduction.MEAN.  Only L1 has a sign mask to impose.

With the default cfg (b1leakyrelu, l1) it is ResOracle, operation for operation.
"""
from collections import OrderedDict

import numpy as np
import torch

import resblock_oracle as R

HUBER_DELTA = 0.1


class OptOracle(R.ResOracle):
    def b1leakyrelu(self, x, b, site=None):
        """The brelu of cfg["activation"] (every caller of b1leakyrelu in the oracles is a brelu site)."""
        act = self.cfg.get("activation", "b1leakyrelu")
        if act == "b1leakyrelu":
            return super().b1leakyrelu(x, b, site)
        if act == "b1relu":
            return self.b1relu(x, b, site)
        if act == "b1tanh":
            return self.b1tanh(x, b)
        raise NotImplementedError(act)

    def recon_loss(self, d):
        """models.py:357-369 on the residual d = x_hat - gt."""
        loss = self.cfg.get("loss", "l1")
        if loss == "l1":
            if self.masks is not None and "l1_sign" in self.masks:
                return (self.masks["l1_sign"].to(d.dtype) * d).mean()
            return d.abs().mean()
        if loss == "huber":
            e = d.abs()
            q = torch.clamp(e, max=HUBER_DELTA)
            return (0.5 * q * q + HUBER_DELTA * (e - q)).mean()
        return (d * d).mean()

    def losses(self, x_hat, gt, z_mean, z_logvar, d_real, d_fake, P, edges, smooth=0.1):
        """Oracle.losses with the configured reconstruction term."""
        cfg = self.cfg
        d = x_hat - gt
        recon = self.recon_loss(d)
        if self.record is not None:
            self.record["l1_sign"] = torch.sign(d.detach())
        latent = (-0.5 * (1 + z_logvar - z_mean ** 2 - torch.exp(z_logvar)).sum(1)).mean()
        e0 = torch.as_tensor(edges[:, 0].astype(np.int64))
        e1 = torch.as_tensor(edges[:, 1].astype(np.int64))
        ev = lambda a: a[:, e0] - a[:, e1]
        edge = torch.linalg.norm(ev(x_hat) - ev(gt), dim=-1).mean()
        reg = cfg["regularization"]
        reg_g = 0.0
        for name in ("generator/encoder/fc_mean", "generator/encoder/fc_var", "generator/decoder/fc1"):
            reg_g = reg_g + reg * (P[name + "/dense/kernel"] ** 2).sum() / 2
        reg_g = reg * reg_g
        out = OrderedDict(recon=recon, latent=latent, edge=edge, reg_g=reg_g)
        if d_fake is not None:
            out["gan_g"] = self.bce_logits(d_fake, 1 - smooth)
            out["loss_g"] = (out["gan_g"] * cfg["lambda_gan"] + recon * cfg["lambda_recon"] + edge * cfg["lambda_edge"]
                             + latent * cfg["lambda_latent"] + reg_g)
            if d_real is not None:
                out["gan_d"] = self.bce_logits(d_real, 1 - smooth) + self.bce_logits(d_fake, smooth)
                out["loss_d"] = out["gan_d"] * cfg["lambda_gan"]
        return out
