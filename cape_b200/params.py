"""Model configuration and parameter inventory, named exactly like the reference's TF variables
(scopes at lib/models.py:162,492-510,539-560,578-616,668-676,748-768,780-789,801) so that a converted
reference checkpoint can be dropped in by name."""
from collections import OrderedDict

import numpy as np

DEFAULTS = dict(
    # architecture (main.py:35-40,60-70; config_parser.py defaults)
    F=[64, 64, 128, 128, 256, 256, 512, 512], K=[2] * 8, Kd=3, nz=18, nz_cond=24, nz_cond2=8,
    cond_dim=126, cond2_dim=4, n_layer_cond=1, reduce_dim=64, affine=False, nn_input_channel=3,
    use_res_block=False, use_res_block_dec=True, cond_encoder=False, optim_condnet=True, activation="b1leakyrelu",
    # optimisation / loss (config_parser.py:27-46)
    lr=8e-3, lr_scaler=0.1, decay_rate=0.99, decay_steps=1, momentum=0.9, lr_warmup=False, optimizer="sgd",
    regularization=2e-3, lambda_recon=1.0, lambda_edge=1.0, lambda_latent=8e-4, lambda_gan=0.1, loss="l1",
    batch_size=16, seed=123,
)

NZ64_AFFINE = dict(DEFAULTS, nz=64, nz_cond=32, nz_cond2=32, affine=True, lr_warmup=True)   # configs/CAPE-affineconv_nz64_*.yaml
NZ18_PLAIN = dict(DEFAULTS, nz=18, nz_cond=24, nz_cond2=8, affine=False, lr_warmup=True)    # configs/CAPE_nz18_*.yaml


def cond_fc1_width(nz_cond, y_dim):
    """Hidden width of the 2-layer condition net (lib/models.py:498-503)."""
    if nz_cond < y_dim // 2:
        return y_dim // 2
    if nz_cond < y_dim * 2:
        return y_dim
    return nz_cond // 2


def param_specs(cfg, p, p_d):
    """Ordered {name: shape}.  p / p_d: vertex counts of the VAE / discriminator hierarchies."""
    F, K, Kd = cfg["F"], cfg["K"], cfg["Kd"]
    nz, nzc, nzc2 = cfg["nz"], cfg["nz_cond"], cfg["nz_cond2"]
    Cc = nzc + nzc2
    s = OrderedDict()
    # condition nets (models.py:479-511; pose net has nlayers=2 hard-coded at :284)
    h = cond_fc1_width(nzc, cfg["cond_dim"])
    s["condition_pose/fc1/dense/kernel"] = (cfg["cond_dim"], h)
    s["condition_pose/fc1/dense/bias"] = (h,)
    s["condition_pose/fc2/dense/kernel"] = (h, nzc)
    s["condition_pose/fc2/dense/bias"] = (nzc,)
    if cfg.get("n_layer_cond", 1) == 1:
        s["condition_clo_label/fc1/dense/kernel"] = (cfg["cond2_dim"], nzc2)
        s["condition_clo_label/fc1/dense/bias"] = (nzc2,)
    else:
        h2 = cond_fc1_width(nzc2, cfg["cond2_dim"])
        s["condition_clo_label/fc1/dense/kernel"] = (cfg["cond2_dim"], h2)
        s["condition_clo_label/fc1/dense/bias"] = (h2,)
        s["condition_clo_label/fc2/dense/kernel"] = (h2, nzc2)
        s["condition_clo_label/fc2/dense/bias"] = (nzc2,)
    # encoder (models.py:514-561); cond_encoder: the first layer also sees [y | y2] on every vertex (:531-535)
    fin = cfg["nn_input_channel"] + (Cc if cfg.get("cond_encoder") else 0)
    for i in range(len(F)):
        if cfg.get("use_res_block"):
            sc = "generator/encoder/encoder_resblock%d" % (i + 1)        # res_block, models.py:715-741
            s[sc + "/filter_1/weights"] = (fin * K[i], F[i])
            s[sc + "/bias_relu_1/bias"] = (1, 1, F[i])
            s[sc + "/filter_2/weights"] = (F[i] * K[i], F[i])
            if fin != F[i]:
                s[sc + "/1x1-conv/weights"] = (fin, F[i])
            s[sc + "/bias_relu_2/bias"] = (1, 1, F[i])
        else:
            s["generator/encoder/encoder_conv%d/weights" % (i + 1)] = (fin * K[i], F[i])
            s["generator/encoder/encoder_conv%d/bias" % (i + 1)] = (1, 1, F[i])
        fin = F[i]
    rd = cfg["reduce_dim"]
    red = F[-1] // (F[-1] // rd) if rd > 0 else F[-1]
    if rd > 0:
        s["generator/encoder/1x1-conv/weights"] = (F[-1], red)
    flat = p[-1] * red
    for n in ("fc_mean", "fc_var"):
        s["generator/encoder/%s/dense/kernel" % n] = (flat, nz)
        s["generator/encoder/%s/dense/bias" % n] = (nz,)
    # decoder (models.py:564-617)
    s["generator/decoder/fc1/dense/kernel"] = (nz + Cc, flat)
    s["generator/decoder/fc1/dense/bias"] = (flat,)
    if rd > 0:
        s["generator/decoder/1x1-conv/weights"] = (red, F[-1])
    fin = F[-1] + Cc
    for i in range(len(F)):
        Fo = F[-i - 1]
        Kb = K[-i - 1]
        if not cfg["use_res_block_dec"]:
            # udn (models.py:173-191, chosen at :597-603 whatever `affine` says): unpool, filter, brelu
            sc = "generator/decoder/decoder_conv%d" % (i + 1)
            s[sc + "/weights"] = (fin * Kb, Fo)
            s[sc + "/bias"] = (1, 1, Fo)
            fin = Fo + Cc
        elif cfg["affine"]:
            sc = "generator/decoder/decoder_resblock_affine%d" % (i + 1)
            s[sc + "/graph_conv/weights"] = (fin * Kb, Fo // 2)
            s[sc + "/affine/weights"] = (fin, Fo // 2)
            fin = Fo // 2 + Cc
        else:
            sc = "generator/decoder/decoder_resblock_cmr%d" % (i + 1)
            s[sc + "/group_norm/gamma"] = (fin,)
            s[sc + "/group_norm/beta"] = (fin,)
            s[sc + "/graph_linear_1/weights"] = (fin, Fo // 2)
            s[sc + "/group_norm_1/gamma"] = (Fo // 2,)
            s[sc + "/group_norm_1/beta"] = (Fo // 2,)
            s[sc + "/graph_conv/weights"] = (Fo // 2 * Kb, Fo // 2)
            s[sc + "/group_norm_2/gamma"] = (Fo // 2,)
            s[sc + "/group_norm_2/beta"] = (Fo // 2,)
            s[sc + "/graph_linear_2/weights"] = (Fo // 2, Fo)
            if fin != Fo:
                s[sc + "/graph_linear_input/weights"] = (fin, Fo)
            fin = Fo + Cc
    s["generator/decoder/outputs/weights"] = (fin * K[0], cfg["nn_input_channel"])
    s["generator/decoder/outputs/bias"] = (1, p[0], cfg["nn_input_channel"])
    # discriminator (models.py:648-678, :796-810)
    fin = cfg["nn_input_channel"] + Cc
    for i in range(len(p_d) - 1):
        s["discriminator/shared/conv%d/weights" % (i + 1)] = (fin * Kd, F[i])
        s["discriminator/shared/conv%d/bias" % (i + 1)] = (1, 1, F[i])
        fin = F[i]
    s["discriminator/prediction_map/weights"] = (fin * K[-1], 1)
    return s


def init_params(specs, seed=123):
    """Reference initialisers: graph-conv weights truncated_normal(0, 0.1) (models.py:217-219), graph-conv
    biases 0.1 (:223-225), dense kernels glorot-uniform / zero bias (tf.layers.dense defaults), GN gamma 1, beta 0
    (:702-703).  Returns {name: float32 ndarray}."""
    rng = np.random.RandomState(seed)
    out = OrderedDict()
    for name, shape in specs.items():
        if name.endswith("dense/kernel"):
            lim = np.sqrt(6.0 / (shape[0] + shape[1]))
            v = rng.uniform(-lim, lim, size=shape)
        elif name.endswith("dense/bias") or name.endswith("/beta"):
            v = np.zeros(shape)
        elif name.endswith("/gamma"):
            v = np.ones(shape)
        elif name.endswith("/bias"):
            v = np.full(shape, 0.1)
        elif name.endswith("/weights"):
            v = rng.normal(0.0, 0.1, size=shape)
            bad = np.abs(v) > 0.2
            while bad.any():                      # truncated normal: resample beyond 2 sigma
                v[bad] = rng.normal(0.0, 0.1, size=int(bad.sum()))
                bad = np.abs(v) > 0.2
        else:
            raise KeyError(name)
        out[name] = v.astype(np.float32)
    return out


def is_g_param(name, optim_condnet=True):
    """Variable filter of CAPE.training (models.py:455-458)."""
    return name.startswith("generator") or (optim_condnet and "condition" in name)


def is_d_param(name):
    return name.startswith("discriminator")
