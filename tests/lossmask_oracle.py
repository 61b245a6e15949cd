"""CPU oracle of the reference's `--loss_mask binary` -- TEST INFRASTRUCTURE ONLY.

`MaskOracle` extends tests/options_oracle.OptOracle with the `weights=self.loss_mask` that lib/models.py:357-369 hands
to every reconstruction loss.  With cfg["loss_mask"] == "binary" the weights are W[n, v, c] = m[v], m the shipped
per-vertex mask (cape_b200.topology.loss_mask_binary), and TF-1's Reduction.MEAN divides the weighted sum by the sum of
the weights broadcast to the loss's shape:

    recon = sum_{n,v,c} m[v] l(d) / sum_{n,v,c} m[v]

Any other value of cfg["loss_mask"] means weights 1.0 (models.py:47-52), and then it is OptOracle, operation for
operation.  The edge, KL, GAN and regularisation terms are OptOracle's.
"""
import torch

import options_oracle as OO
from cape_b200 import topology as T


def weights(d):
    """The [1, rows, 1] weights of the residual d [N, rows, 3], in d's dtype."""
    return torch.as_tensor(T.loss_mask_binary(), dtype=d.dtype)[None, :, None]


def recon_terms(loss, d, sign=None):
    """Per-coordinate reconstruction loss of models.py:357-369 on the residual d; sign: an imposed sign(d) for L1."""
    if loss == "l1":
        return sign.to(d.dtype) * d if sign is not None else d.abs()
    if loss == "huber":
        e = d.abs()
        q = torch.clamp(e, max=OO.HUBER_DELTA)
        return 0.5 * q * q + OO.HUBER_DELTA * (e - q)
    return d * d


class MaskOracle(OO.OptOracle):
    def recon_loss(self, d):
        if self.cfg.get("loss_mask") != "binary":
            return super().recon_loss(d)
        sign = self.masks.get("l1_sign") if self.masks is not None else None
        w = weights(d)
        return (recon_terms(self.cfg.get("loss", "l1"), d, sign) * w).sum() / (torch.ones_like(d) * w).sum()
