"""`CAPE`: the reference's model class (lib/models.py:230-1174) on top of the H100 kernels.

Same constructor keywords as `models.CAPE(L=, D=, U=, L_d=, D_d=, **params)` built by main.py:50-87, same
public methods (`build_graph`, `fit`, `encode`, `encode_only_condition`, `predict`, `evaluate`, `decode`,
`get_var`) with the same argument meaning, numpy in / numpy out, static batch size with zero padding of the
last batch (lib/models.py:945-953,1046-1050).  There is no TF session: `build_graph` allocates the device
buffers and weights, checkpoints are .npz files keyed by the reference's TF variable names.
"""
import collections
import os
import time

import numpy as np
import torch

from . import _lib
from . import engine as E
from . import summary as S
from .network import CapeNetwork
from .params import DEFAULTS


class CAPE(object):
    def __init__(self, L, D, U, L_d, D_d, lr_scaler, lambda_gan, use_res_block, use_res_block_dec, nz_cond2,
                 cond2_dim, Kd, n_layer_cond=1, cond_encoder=True, reduce_dim=True, affine=False, lr_warmup=False,
                 optim_condnet=True, F=None, K=None, p=None, nz=18, loss="l1", nn_input_channel=3,
                 filter="chebyshev5", activation="b1leakyrelu", pool="poolwT", unpool="poolwT", num_epochs=60,
                 lr=0.008, decay_rate=0.99, optimizer="sgd", decay_steps=None, momentum=0.9, cond_dim=0, nz_cond=0,
                 regularization=0, batch_size=32, seed=123, lambda_recon=1.0, lambda_edge=0.0, lambda_latent=1e-3,
                 restart=False, name="", loss_mask=None, device=0, ref_compat=True, checkpoint_dir="checkpoints",
                 device_dataset=True, summary_dir=None, **unused):
        # name-based operator seam of base_model (lib/models.py:58-62): kernels exist for chebyshev5 / poolwT and the
        # one-bias-per-filter activations
        if (filter, pool, unpool) != ("chebyshev5", "poolwT", "poolwT"):
            raise NotImplementedError("kernels exist for filter='chebyshev5' and pool=unpool='poolwT' (the configuration "
                                      "of every shipped config)")
        E.brelu(activation)                  # b1leakyrelu, b1relu or b1tanh; anything else raises
        self.Laplacian, self.Downsample_mtx, self.Upsample_mtx, self.p = L, D, U, p
        self.Laplacian_d, self.Downsample_mtx_d = L_d, D_d
        self.input_num_verts = L[0].shape[0]
        self.nn_input_channel = nn_input_channel
        self.name, self.restart = name, restart
        self.batch_size, self.num_epochs = int(batch_size), num_epochs
        self.nz, self.nz_cond, self.nz_cond2 = int(nz), nz_cond, nz_cond2
        self.cond_dim, self.cond2_dim = cond_dim, cond2_dim
        self.lambda_l1, self.lambda_edge, self.lambda_latent = lambda_recon, lambda_edge, lambda_latent
        self.device_index, self.ref_compat, self.checkpoint_dir = device, ref_compat, checkpoint_dir
        self.device_dataset = bool(device_dataset)
        # TensorBoard summaries of `fit` under <summary_dir>/<name> (the reference's `summaries` folder); None: none
        self.summary_dir = summary_dir
        rd = reduce_dim if not isinstance(reduce_dim, bool) else (64 if reduce_dim else 0)
        if rd < 0:
            raise ValueError("reduce dim must be greater than 0!")           # lib/models.py:259
        self.cfg = dict(DEFAULTS, F=list(F), K=list(K), Kd=Kd, nz=int(nz), nz_cond=nz_cond, nz_cond2=nz_cond2,
                        cond_dim=cond_dim, cond2_dim=cond2_dim, n_layer_cond=n_layer_cond, reduce_dim=rd,
                        affine=bool(affine), nn_input_channel=nn_input_channel, use_res_block=bool(use_res_block),
                        use_res_block_dec=bool(use_res_block_dec), cond_encoder=bool(cond_encoder),
                        optim_condnet=bool(optim_condnet), lr=lr, lr_scaler=lr_scaler, decay_rate=decay_rate,
                        decay_steps=decay_steps if decay_steps else 1, momentum=momentum, lr_warmup=bool(lr_warmup),
                        optimizer=optimizer, regularization=regularization, lambda_recon=lambda_recon,
                        lambda_edge=lambda_edge, lambda_latent=lambda_latent, lambda_gan=lambda_gan, loss=loss,
                        activation=activation, loss_mask=loss_mask if loss_mask == "binary" else None,
                        batch_size=int(batch_size), seed=seed)
        self.net = None
        self.rng = np.random.RandomState(seed)
        self.global_step = 0
        # where the current weights come from: "init" (random initialisers), "checkpoint", "fit", "set"
        self._weights_source = "init"

    # ---- graph -------------------------------------------------------------------------------------------
    def build_graph(self, input_num_verts, nn_input_channel, phase="train"):
        """Allocate weights/buffers (reference: lib/models.py:267-351).  `phase` is accepted for compatibility: the
        same engine serves training and the demo-time encode/decode entry points."""
        assert input_num_verts == self.input_num_verts and nn_input_channel == self.nn_input_channel
        if self.net is None:
            self.net = CapeNetwork(self.Laplacian, self.Downsample_mtx, self.Upsample_mtx, self.Laplacian_d,
                                   self.Downsample_mtx_d, self.cfg, self.batch_size, device=self.device_index,
                                   ref_compat=self.ref_compat)
        self.phase = phase
        return self

    def _get_path(self, folder):
        """<folder>/<experiment name> (lib/models.py:204-207); config_parser's default name is None -> no sub-folder."""
        name = self.name if self.name is not None else ""
        if not isinstance(name, str):
            raise ValueError("experiment name must be a string, got %r" % (name,))
        return os.path.join(folder, name)

    def _get_session(self, sess=None):
        """The reference's inference entry points open a session and restore the newest checkpoint when none is
        passed (lib/models.py:209-215, 941, 1040, 1140); with no TF session here, "restoring" happens once: weights
        that are still the random initialisers are replaced by the newest checkpoint, and a missing checkpoint is an
        error instead of a silent run on random weights.  A non-None `sess`, `fit`, `restore` or `load_weights`
        count as "the caller has put weights in place"."""
        if sess is None and self._weights_source == "init":
            self.restore()
        return self

    def load_weights(self, values):
        """Set all weights from {TF variable name: array} (e.g. cape_b200.tf_checkpoint.read_checkpoint)."""
        self.net.set_params(values)
        self._weights_source = "set"

    def save(self, step):
        path = self._get_path(self.checkpoint_dir)
        os.makedirs(path, exist_ok=True)
        vals = self.net.get_params()
        mom = {"momentum/" + k: v for k, v in {**self.net.PG.export(self.net.PG.mom),
                                                **self.net.PD.export(self.net.PD.mom)}.items()}
        if self.net.adam:            # second-moment slots and the application count (TF: beta1_power = 0.9 ** (t + 1))
            mom.update({"adam_v/" + k: v for k, v in {**self.net.PG.export(self.net.PG.var),
                                                       **self.net.PD.export(self.net.PD.var)}.items()})
            mom["adam_t"] = np.int64(self.net.adam_t)
        fn = os.path.join(path, "model-%d.npz" % step)
        np.savez(fn, global_step=np.int64(self.global_step), **vals, **mom)
        return fn

    def save_tf(self, step):
        """Write the weights as a TensorFlow V2 checkpoint `model.ckpt-<step>` (the reference's tf.train.Saver format,
        lib/models.py:351,923-924: variables by name, optimiser slots as `<variable>/Momentum`, `global_step`) so
        that they can be handed back to the reference."""
        from . import tf_checkpoint
        path = self._get_path(self.checkpoint_dir)
        vals = dict(self.net.get_params())
        slot = "/Adam" if self.net.adam else "/Momentum"     # slot names of tf.train.AdamOptimizer / MomentumOptimizer
        for k, v in {**self.net.PG.export(self.net.PG.mom), **self.net.PD.export(self.net.PD.mom)}.items():
            vals[k + slot] = v
        if self.net.adam:
            from .network import ADAM_BETA1, ADAM_BETA2
            for k, v in {**self.net.PG.export(self.net.PG.var), **self.net.PD.export(self.net.PD.var)}.items():
                vals[k + "/Adam_1"] = v
            t1 = self.net.adam_t + 1
            for sfx in ("", "_1"):                           # opt_g's and opt_d's non-slot variables
                vals["beta1_power" + sfx] = np.asarray(ADAM_BETA1 ** t1, np.float32)
                vals["beta2_power" + sfx] = np.asarray(ADAM_BETA2 ** t1, np.float32)
        vals["global_step"] = np.asarray(self.global_step, np.int64)
        return tf_checkpoint.write_checkpoint(os.path.join(path, "model.ckpt-%d" % step), vals)

    def restore(self, filename=None):
        """Load the newest checkpoint of this run (reference: _get_session, lib/models.py:209-215): a `.npz` written
        by `save`, or a TensorFlow checkpoint prefix (`model.ckpt-N`: the reference's own / published models,
        README.md:104) read by cape_b200.tf_checkpoint -- the parameter names are the reference's variable names."""
        from . import tf_checkpoint
        path = self._get_path(self.checkpoint_dir)
        if filename is None:
            cands = sorted((f for f in os.listdir(path) if f.startswith("model-") and f.endswith(".npz")),
                           key=lambda f: int(f[6:-4])) if os.path.isdir(path) else []
            if cands:
                filename = os.path.join(path, cands[-1])
            else:
                filename = tf_checkpoint.latest_checkpoint(path) if os.path.isdir(path) else None
            if filename is None:
                raise FileNotFoundError("no checkpoint under %s" % path)
        adam = self.net.adam
        if tf_checkpoint.is_checkpoint(filename):
            z = tf_checkpoint.read_checkpoint(filename)
            files, mom_key = list(z), (lambda n: n + ("/Adam" if adam else "/Momentum"))
            var_key = lambda n: n + "/Adam_1"
            if adam and "beta1_power" in files:
                from .network import ADAM_BETA1
                self.net.adam_t = max(int(round(np.log(float(z["beta1_power"])) / np.log(ADAM_BETA1))) - 1, 0)
        else:
            z = np.load(filename)
            files, mom_key = z.files, (lambda n: "momentum/" + n)
            var_key = lambda n: "adam_v/" + n
            if adam and "adam_t" in files:
                self.net.adam_t = int(z["adam_t"])
        want = set(self.net.PG.names) | set(self.net.PD.names)
        missing = sorted(want - set(files))
        if missing:
            raise KeyError("checkpoint %s lacks %d variables of this architecture, e.g. %s" % (filename, len(missing),
                                                                                        missing[:3]))
        self.net.set_params({k: np.asarray(z[k]).reshape(self.net.specs[k]) for k in want})
        for P in (self.net.PG, self.net.PD):
            for n in P.names:
                if mom_key(n) in files:
                    P._view(P.mom, n).copy_(torch.as_tensor(np.asarray(z[mom_key(n)], np.float32).reshape(-1)))
                if adam and var_key(n) in files:
                    P._view(P.var, n).copy_(torch.as_tensor(np.asarray(z[var_key(n)], np.float32).reshape(-1)))
        self.global_step = int(z["global_step"]) if "global_step" in files else 0
        self._weights_source = "checkpoint"
        return filename

    def get_var(self, name):
        return self.net.get_params()[name]

    # ---- helpers ------------------------------------------------------------------------------------------
    def _pad(self, a, width=None):
        a = np.asarray(a, np.float32)
        out = np.zeros((self.batch_size,) + a.shape[1:], np.float32)
        out[: a.shape[0]] = a
        return torch.from_numpy(out)

    def _stage_g(self, data=None, cond=None, cond2=None, eps=None):
        net, N = self.net, self.batch_size
        if data is not None:
            net.in_x.copy_(self._pad(data))
        if cond is not None:
            net.in_cond[N:].copy_(self._pad(cond))
            net.in_cond2[N:].copy_(self._pad(cond2))
        if eps is not None:
            net.in_eps.copy_(torch.from_numpy(np.asarray(eps, np.float32)))

    # ---- training (lib/models.py:837-929) ---------------------------------------------------------------------
    def fit(self, data_wrapper):
        """Training loop of lib/models.py:837-929.  Two things differ from the reference, neither visible in the
        results: the training split is uploaded to the GPU once and every batch is assembled there from indices
        (load_data.DeviceDataset; `device_dataset=False` keeps the host path), and under torch.distributed (launch with
        torchrun, one process per GPU) every rank trains on its own `batch_size` meshes per update with the gradients
        averaged over ranks (cape_b200.distributed) -- weights stay identical on all ranks, rank 0 validates and saves."""
        from . import distributed as DP
        from .load_data import DeviceDataset
        import torch.distributed as dist
        train_data, train_cond, train_cond2 = data_wrapper.vertices_train, data_wrapper.cond1_train, data_wrapper.cond2_train
        val = (data_wrapper.vertices_val, data_wrapper.cond1_val, data_wrapper.cond2_val, data_wrapper.vertices_val)
        N = self.batch_size
        num_steps_epoch = int(train_data.shape[0] / N)
        num_steps = self.num_epochs * num_steps_epoch
        t_start = time.time()
        if self.restart is not True:
            self.restore()
            start_step = self.global_step
        else:
            if not self.name:
                raise ValueError("Please provide an expriment name by setting the --name flag.")   # models.py:858-859
            start_step, self.global_step = 1, 0
        self._weights_source = "fit"
        net = self.net
        rank, world = (dist.get_rank(), dist.get_world_size()) if dist.is_available() and dist.is_initialized() else (0, 1)
        allreduce = DP.make_allreduce(world)
        if world > 1:
            DP.broadcast_params([net.PG.flat, net.PD.flat, net.PG.mom, net.PD.mom])
            net.prep_weights()
            draw = np.random.RandomState(DP.rank_seed(self.cfg["seed"], rank))       # every rank its own batches / noise
            self.rng = np.random.RandomState(DP.rank_seed(self.cfg["seed"] + 1, rank))
        else:
            draw = np.random                                                            # the reference's global stream
        dev = None
        if self.device_dataset:
            dev = DeviceDataset(train_data, train_cond, train_cond2, net.device)
        writer = self._open_summaries() if (self.summary_dir is not None and rank == 0) else None
        losses = []
        indices_g, indices_d = collections.deque(), collections.deque()
        for step in range(start_step, start_step + num_steps):
            if len(indices_g) < N:
                indices_g.extend(draw.permutation(train_data.shape[0]))
            if len(indices_d) < N:
                indices_d.extend(draw.permutation(train_data.shape[0]))
            idx_g = [indices_g.popleft() for _ in range(N)]
            idx_d = [indices_d.popleft() for _ in range(N)]
            t = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float32))
            # the reference runs the G+D update twice per loop step (both op_train_* depend on both apply ops,
            # models.py:470-472,905-906), each with fresh eps; ref_compat keeps that, otherwise one update per step
            for _ in range(2 if self.ref_compat else 1):
                eps = self.rng.normal(size=(N, self.nz)).astype(np.float32)
                if dev is not None:
                    dev.stage(net, idx_g, idx_d, eps)
                else:
                    net.set_inputs(t(train_data[idx_g]), t(train_cond[idx_g]), t(train_cond2[idx_g]), t(eps),
                                   t(train_data[idx_d]), t(train_cond[idx_d]), t(train_cond2[idx_d]))
                # both apply_gradients share global_step (models.py:462,467): it advances by 2 per update
                net.train_step(step=self.global_step, allreduce=allreduce)
                self.global_step += 2
            if (step % num_steps_epoch == 0 or step == num_steps) and rank == 0:
                summary = self._summary_values() if writer is not None else None
                string, recon, latent, edge = self.evaluate(*val)
                losses.append(recon)
                print("step {} / {}: validation {}  time: {:.0f}s".format(step, num_steps, string, time.time() - t_start))
                if writer is not None:
                    scalars, histograms = summary
                    writer.add(step, scalars + [(S.VALIDATION_TAG, recon)], histograms)
                self.save(step)
        if writer is not None:
            writer.close()
        t_step = (time.time() - t_start) / max(num_steps, 1)
        return losses, t_step

    # ---- TensorBoard summaries (lib/models.py:868,919-922) -------------------------------------------------------------
    def _open_summaries(self):
        """A new event file in <summary_dir>/<name>.  At restart the reference deletes that folder (models.py:861); here
        only the event files directly in it go.  The moving averages start at 0 with every `fit`."""
        path = self._get_path(self.summary_dir)
        if self.restart is True:
            S.remove_event_files(path)
        self.net.track_loss_average()
        # the summary pass's own noise: training draws exactly what it draws without summaries
        self._summary_rng = np.random.RandomState(self.cfg["seed"])
        return S.EventWriter(path)

    def _summary_values(self):
        """sess.run(op_summary) on the loop step's batch (models.py:919): one more forward pass of both players at the
        updated weights with fresh noise, no training op.  Returns ([(tag, value)], [(tag, HistogramProto bytes)])."""
        net, c = self.net, self.cfg
        eps = self._summary_rng.normal(size=(self.batch_size, self.nz)).astype(np.float32)
        net.in_eps.copy_(torch.from_numpy(eps))
        net.enqueue_loss_forward()
        net.enqueue_fc_sumsq()
        hist = net.weight_histograms()
        v = net.losses.cpu().numpy()
        avg = net.loss_avg.cpu().numpy()
        f32 = np.float32
        r = f32(c["regularization"])
        reg_g = r * (r * (net.fc_sumsq.cpu().numpy()[0] * f32(0.5)))       # r * sum_W r * l2_loss(W), as cape_loss_ema
        lr_g, lr_d = net.lr_now(self.global_step)
        scalars = list(zip(S.SCALAR_TAGS, [v[0], v[2], reg_g, 0.0, v[3], v[4] + v[5], avg[0], avg[1], lr_g, lr_d]))
        limits = S.bucket_limits()
        histograms = []
        for name in net.histogram_names():
            stats, nonfinite, counts = hist[name]
            if nonfinite:
                raise ValueError("Nan in summary histogram for: %s" % name)
            histograms.append((name, S.encode_histogram(stats, counts, limits)))
        return scalars, histograms

    # ---- inference entry points (lib/models.py:931-1174) --------------------------------------------------------
    def encode(self, data=None, cond=None, cond2=None):
        self._get_session(None)
        size, N, net = data.shape[0], self.batch_size, self.net
        zm, zl = np.zeros((size, self.nz), np.float32), np.zeros((size, self.nz), np.float32)
        zc = np.zeros((size, self.nz_cond), np.float32)
        zc2 = np.zeros((size, self.nz_cond2), np.float32)
        for b in range(0, size, N):
            e = min(b + N, size)
            self._stage_g(data[b:e], cond[b:e], cond2[b:e])
            net.cond_fwd(N, 2 * N)
            net.encoder_fwd()
            y = net.ycat_g.cpu().numpy()
            zm[b:e], zl[b:e] = net.z_mean.cpu().numpy()[: e - b], net.z_logvar.cpu().numpy()[: e - b]
            zc[b:e], zc2[b:e] = y[: e - b, : self.nz_cond], y[: e - b, self.nz_cond:]
        return zm, zl, zc, zc2

    def encode_only_condition(self, cond=None, cond2=None):
        self._get_session(None)
        size, N, net = cond.shape[0], self.batch_size, self.net
        zc = np.zeros((size, self.nz_cond), np.float32)
        zc2 = np.zeros((size, self.nz_cond2), np.float32)
        for b in range(0, size, N):
            e = min(b + N, size)
            self._stage_g(None, cond[b:e], cond2[b:e])
            net.cond_fwd(N, 2 * N)
            y = net.ycat_g.cpu().numpy()
            zc[b:e], zc2[b:e] = y[: e - b, : self.nz_cond], y[: e - b, self.nz_cond:]
        return zc, zc2

    def predict(self, data, cond=None, cond2=None, labels=None, sess=None, phase="train"):
        self._get_session(sess)
        size, N, net = data.shape[0], self.batch_size, self.net
        preds = np.zeros((size,) + data.shape[1:], np.float32)
        lr_, ll_, le_ = [], [], []
        # reference quirk: true division makes this equal batch_size, so the last batch gets weight 0 (models.py:1039)
        num_zero_phs = N * (size / N + 1) - size
        for b in range(0, size, N):
            e = min(b + N, size)
            eps = self.rng.normal(size=(N, self.nz)).astype(np.float32)      # vae_sampling draws eps at test time too
            self._stage_g(data[b:e], cond[b:e], cond2[b:e], eps)
            net.forward_generator()
            preds[b:e] = net.x_hat.cpu().numpy()[: e - b]
            if labels is not None:
                gt = self._pad(labels[b:e]).to(net.device)
                net.losses.zero_()
                kind = E.recon_kind(self.cfg["loss"])               # the configured loss (models.py:357-369)
                rest = (net.n_edges, E._ptr(net.z_mean), E._ptr(net.z_logvar), self.nz, E._ptr(net.d_xhat),
                      E._ptr(net.losses), E._stream())
                if self.cfg["loss_mask"] == "binary":
                    # the masked term (models.py:1073), the mask covering the whole zero-padded batch
                    E.recon_losses(net.tp, net.nbr_op, net.x_hat, gt, N, net.p[0], kind, 0.0, 0.0, net.n_edges,
                                   net.z_mean, net.z_logvar, self.nz, net.d_xhat, net.losses, mask=net.loss_mask,
                                   mask_sum=net.loss_mask_sum)
                    rc = 0
                elif kind == E.RECON_L1:
                    rc = net.tp.lib.cape_recon_losses(net.tp.h, net.nbr_op, E._ptr(net.x_hat), E._ptr(gt), N, net.p[0],
                                                      0.0, 0.0, *rest)
                else:
                    rc = net.tp.lib.cape_recon_losses_ex(net.tp.h, net.nbr_op, E._ptr(net.x_hat), E._ptr(gt), N,
                                                         net.p[0], kind, E.HUBER_DELTA, 0.0, 0.0, *rest)
                _lib.check(rc)
                v = net.losses.cpu().numpy()
                lr_.append(v[0]); le_.append(v[1]); ll_.append(v[2])
        if labels is None:
            return preds

        def calc_mean(c):
            return (np.sum(np.array(c)[:-1]) * N + c[-1] * (N - num_zero_phs)) / size      # models.py:1083-1086

        return preds, calc_mean(lr_), calc_mean(ll_), calc_mean(le_)

    def evaluate(self, data, cond=None, cond2=None, labels=None, sess=None):
        t0 = time.time()
        _, recon, latent, edge = self.predict(data, cond, cond2, labels, sess)
        s = "recon loss: {:.2e}, latent loss: {:.2e}, edge_loss: {:.2e}(weighted)".format(
            recon * self.lambda_l1, latent * self.lambda_latent, edge * self.lambda_edge)
        if sess is None:
            s += "\ntime: {:.0f}s".format(time.time() - t0)
        return s, recon, latent, edge

    def decode(self, data, cond=None, cond2=None):
        """data: z_total [size, nz+nz_cond+nz_cond2]; cond / cond2: condition EMBEDDINGS (lib/models.py:1128-1174);
        a single condition row is broadcast over the batch as in the demos (:1152-1153)."""
        self._get_session(None)
        size, N, net = data.shape[0], self.batch_size, self.net
        x_rec = np.zeros((size, self.input_num_verts, self.nn_input_channel), np.float32)
        for b in range(0, size, N):
            e = min(b + N, size)
            zt = self._pad(data[b:e]).to(net.device)
            if cond.shape[0] == 1:
                c1, c2 = np.repeat(cond, e - b, 0), np.repeat(cond2, e - b, 0)
            else:
                c1, c2 = cond[b:e], cond2[b:e]
            yc = self._pad(np.concatenate([c1, c2], 1)).to(net.device)
            out = torch.empty(N, self.input_num_verts, self.nn_input_channel, device=net.device)
            net.decoder_fwd(zt, yc, out)
            x_rec[b:e] = out.cpu().numpy()[: e - b]
        return x_rec
