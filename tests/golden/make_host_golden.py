#!/usr/bin/env python
"""Golden data for the host-side tests that compare with the REFERENCE's own Python (tests/test_reference_golden.py,
tests/test_config.py).  Runs only where a reference checkout exists ($CAPE_REFERENCE); the tests read what it wrote:

  * host_golden.npz -- what the reference's code returns for the stand-in inputs defined here: `BodyData` splits and
    statistics, the meshes `demo_simple` writes (every DEMO_STRIDE-th vertex), the batch streams of `fit`, the results
    of `predict` / `evaluate` / `encode` / `encode_only_condition` / `decode`, the learning rates of `training()`, the
    flags `parse_config` declares and the arguments `models.CAPE` accepts;
  * ref_configs.npz -- the text of the reference's configs/*.yaml.

The inputs and stand-ins live in this file and are imported by the tests, so both sides see the same ones.

    CAPE_REFERENCE=/path/to/CAPE python tests/golden/make_host_golden.py
"""
import argparse
import contextlib
import importlib.util
import inspect
import io
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "host_golden.npz")
CONFIGS_OUT = os.path.join(HERE, "ref_configs.npz")
DEMO_STRIDE = 7                       # vertices kept of every mesh demo_simple writes
PRED_STRIDE = 13                      # entries kept of the [5, 6890, 3] predict / decode results
STUBBED = ("tensorflow", "tensorflow.python", "tensorflow.python.util", "trimesh", "psbody", "psbody.mesh", "smplx")
LR_STEPS = (0, 1, 40, 79, 80, 81, 89, 90, 100, 1234)
FIT_N, FIT_NTRAIN = 2, 7


# ---------------------------------------------------------------------------------------------------------------
# inputs and stand-ins shared by the reference side (here) and our side (the tests)
# ---------------------------------------------------------------------------------------------------------------
def body_data_files(dirname):
    rng = np.random.RandomState(0)
    files = {}
    for split, n in (("train", 37), ("test", 9)):
        files[split + "_disp"] = rng.normal(size=(n, 53, 3)) * 0.01 + rng.normal(size=(1, 53, 3))
        files[split + "_pose"] = rng.normal(size=(n, 72))                     # full poses: filtered to 14 joints
        files[split + "_clo"] = np.eye(4)[rng.randint(0, 4, size=n)]
    fn = {}
    for k, v in files.items():
        fn[k] = os.path.join(str(dirname), k + ".npy")
        np.save(fn[k], v)
    return dict(nVal=5, train_mesh_fn=fn["train_disp"], train_cond1_fn=fn["train_pose"], train_cond2_fn=fn["train_clo"],
                test_mesh_fn=fn["test_disp"], test_cond1_fn=fn["test_pose"], test_cond2_fn=fn["test_clo"])


BODY_KEYS = ("vertices_train", "vertices_val", "vertices_test", "cond1_train", "cond1_val", "cond1_test", "cond2_train",
             "cond2_val", "cond2_test", "mean", "std", "cond1_train_full", "cond1_test_full")


class FakeModel(object):
    """A deterministic stand-in with the three members demo_simple touches (nz, encode_only_condition, decode)."""
    nz = 64

    def encode_only_condition(self, cond, cond2):
        c, c2 = np.asarray(cond, np.float64), np.asarray(cond2, np.float64)
        return np.tanh(c[:, :32] * 3 + 0.1).astype(np.float32), (c2 @ np.linspace(-1, 1, 4 * 32).reshape(4, 32)).astype(np.float32)

    def decode(self, data, cond=None, cond2=None):
        z = np.asarray(data, np.float64)
        basis = np.cos(np.arange(z.shape[1])[:, None] * 0.37 + np.arange(6890 * 3)[None, :] * 0.011)
        return (z @ basis / 8.0 + float(cond.sum()) * 0.01 - float(cond2.sum()) * 0.02).reshape(-1, 6890, 3).astype(np.float32)


def fit_data():
    rng = np.random.RandomState(5)
    n = FIT_NTRAIN
    return types.SimpleNamespace(
        vertices_train=rng.normal(size=(n, 6890, 3)).astype(np.float32),
        cond1_train=rng.normal(size=(n, 126)).astype(np.float32),
        cond2_train=np.eye(4, dtype=np.float32)[rng.randint(0, 4, size=n)],
        vertices_val=rng.normal(size=(3, 6890, 3)).astype(np.float32), cond1_val=rng.normal(size=(3, 126)).astype(np.float32),
        cond2_val=np.eye(4, dtype=np.float32)[rng.randint(0, 4, size=3)])


def fit_stream(log, data):
    """A logged training loop as arrays: event kinds, checkpoint steps, and per optimiser run the training-set rows
    behind x_g / x_d plus the fed condition arrays."""
    kinds = np.array([e[0] for e in log])
    saves = np.array([e[1] for e in log if e[0] == "save"], np.int64)
    runs = [e[1] for e in log if e[0] == "run"]

    def rows(x):
        return [int(np.flatnonzero((data.vertices_train == r).all(axis=(1, 2)))[0]) for r in x]
    out = {"kinds": kinds, "saves": saves, "x_g_rows": np.array([rows(r["x_g"]) for r in runs], np.int64),
           "x_d_rows": np.array([rows(r["x_d"]) for r in runs], np.int64)}
    for k in ("cond_g", "cond2_g", "cond_d", "cond2_d"):
        out[k] = np.stack([np.asarray(r[k], np.float32) for r in runs])
    return out


def predict_inputs():
    rng = np.random.RandomState(9)
    size = 5
    data = rng.normal(size=(size, 6890, 3)).astype(np.float32)
    cond = rng.normal(size=(size, 126)).astype(np.float32)
    cond2 = np.eye(4, dtype=np.float32)[rng.randint(0, 4, size=size)]
    labels = rng.normal(size=(size, 6890, 3)).astype(np.float32)
    return data, cond, cond2, labels


def predict_out(x, c):                  # stand-in network
    return (np.tanh(x) * 0.5 + float(c.sum()) * 1e-3).astype(np.float32)


def predict_losses(x):                  # stand-in recon / latent / edge
    return float(np.abs(x).mean()), float((x ** 2).mean()), float(x.max())


def encdec_inputs():
    rng = np.random.RandomState(4)
    size = 5
    data = rng.normal(size=(size, 6890, 3)).astype(np.float32)
    cond = rng.normal(size=(size, 126)).astype(np.float32)
    cond2 = np.eye(4, dtype=np.float32)[rng.randint(0, 4, size=size)]
    zt = rng.normal(size=(size, 128)).astype(np.float32)
    ye, y2e = rng.normal(size=(1, 32)).astype(np.float32), rng.normal(size=(1, 32)).astype(np.float32)
    return data, cond, cond2, zt, ye, y2e


def f_mean(x):
    return x[:, :64, 0].astype(np.float32) * 2


def f_var(x):
    return x[:, 64:128, 1].astype(np.float32) - 1


def f_c(c):
    return np.tanh(c[:, :32]).astype(np.float32)


def f_c2(c2):
    return (c2 @ np.linspace(0, 1, 128).reshape(4, 32)).astype(np.float32)


def f_dec(z, y, y2):
    return (np.tanh(z[:, :3])[:, None, :] * np.ones((1, 6890, 1)) + (y.sum(1) - y2.sum(1))[:, None, None] * 1e-2
            ).astype(np.float32)


def lr_configs():
    return [dict(lr=8e-3, lr_scaler=0.1, decay_steps=10, decay_rate=0.99, lr_warmup=warm) for warm in (True, False)]


# ---------------------------------------------------------------------------------------------------------------
# the reference side
# ---------------------------------------------------------------------------------------------------------------
@contextlib.contextmanager
def _stubs():
    saved = {k: sys.modules.get(k) for k in STUBBED}
    for k in [k for k in sys.modules if k == "lib" or k.startswith("lib.")]:
        del sys.modules[k]                # the reference's modules bind the stubs installed when they are imported
    try:
        yield
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


def ref_constructor(G, h):
    from cape_b200.config_parser import model_params, parse_config
    from oracle import tf1_shim as S
    out = {}
    with _stubs():
        S.install()
        from lib import models as RM
        # CAPE.__init__ hands **kwargs to its base class: the accepted names are those of both constructors
        names = set()
        for cls in (RM.CAPE, RM.CAPE.__mro__[1]):
            names |= {n for n, q in inspect.signature(cls.__init__).parameters.items()
                      if n != "self" and q.kind != inspect.Parameter.VAR_KEYWORD}
        out["ctor/args"] = np.array(sorted(names))
        yml = os.path.join(G.REF, "configs", "CAPE-affineconv_nz64_pose32_clotype32_male.yaml")
        args, _ = parse_config(["--config", yml, "--mode", "demo"])
        kw = model_params(args)
        kw["p"] = h["p"]
        S.reset()
        with contextlib.redirect_stdout(io.StringIO()):
            m = RM.CAPE(L=h["L"], D=h["D"], U=h["U"], L_d=h["L_d"], D_d=h["D_d"], **kw)
        out["ctor/nz"], out["ctor/affine"], out["ctor/batch_size"] = np.int64(m.nz), np.int64(m.affine), np.int64(m.batch_size)
    return out


def ref_body_data(G, tmp):
    from oracle import tf1_shim as S
    with _stubs():
        S.install()
        from lib import load_data as RL
        args = body_data_files(tmp)
        with contextlib.redirect_stdout(io.StringIO()):
            ref = RL.BodyData(reference_mesh_file="unused.obj", **args)
        return {"bodydata/" + k: getattr(ref, k) for k in BODY_KEYS} | {"bodydata/n_vertex": np.int64(ref.n_vertex)}


def ref_demo_simple(G, tmp):
    from cape_b200 import demos as ours
    from cape_b200 import topology
    from oracle import tf1_shim as S
    with _stubs():
        S.install()
        v, f = topology.template_mesh()

        class _Tri(object):
            def __init__(self, vertices=None, faces=None):
                self.vertices, self.faces = vertices, faces

            def export(self, path):
                ours.write_obj(path, self.vertices, self.faces)

        sys.modules["trimesh"] = types.ModuleType("trimesh")
        sys.modules["trimesh"].load = lambda *a, **k: _Tri(np.asarray(v), np.asarray(f))
        sys.modules["trimesh"].Trimesh = _Tri
        scratch = os.path.join(tmp, "ref")
        os.makedirs(scratch)
        os.symlink(os.path.join(G.REF, "data"), os.path.join(scratch, "data"))
        spec = importlib.util.spec_from_file_location("ref_demos", os.path.join(G.REF, "demos.py"))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        mod.__file__ = os.path.join(scratch, "demos.py")
        with contextlib.redirect_stdout(io.StringIO()):
            ref = mod.demo_simple(FakeModel(), "x", 123)
            ref.sample_vary_clotype()
        files = sorted(os.listdir(ref.results_dir))
        out = {"demo/files": np.array(files)}
        faces = None
        verts = []
        for fn in files:
            rv, rf = ours.read_obj(os.path.join(ref.results_dir, fn))
            assert faces is None or np.array_equal(faces, rf)
            faces = rf
            verts.append(rv[::DEMO_STRIDE].astype(np.float32))
        out["demo/faces"], out["demo/vertices"] = np.asarray(faces, np.int32), np.stack(verts)
        return out


def _shim_feeds(G, cfg, h, N, demo=False):
    params, batch = G.inputs(cfg, h, N)
    feeds = dict(data_g=batch["x_g"], data_d=batch["x_d"], condition_g=batch["cond_g"], condition2_g=batch["cond2_g"],
                 condition_d=batch["cond_d"], condition2_d=batch["cond2_d"], gt=batch["gt"], eps=batch["eps"])
    if demo:
        feeds.update(G.demo_feeds(cfg, N))
    return params, feeds


def ref_fit(G, h, tmp):
    from oracle import tf1_shim as S
    data = fit_data()
    N = FIT_N
    ref_log = []
    with _stubs():
        tag, cfg, _, step = G.configs()[0]
        params, feeds = _shim_feeds(G, cfg, h, N)
        holder = {}

        class Session(object):
            def __init__(self, *a, **k):
                pass

            def run(self, fetches, feed_dict=None):
                model = holder["model"]
                if isinstance(fetches, list) and len(fetches) == 2:               # one optimiser run of the training loop
                    by_name = {id(model.ph_data_g): "x_g", id(model.ph_data_d): "x_d", id(model.ph_cond_g): "cond_g",
                               id(model.ph_cond2_g): "cond2_g", id(model.ph_cond_d): "cond_d", id(model.ph_cond2_d): "cond2_d"}
                    ref_log.append(("run", {by_name[id(k)]: np.asarray(v) for k, v in feed_dict.items() if id(k) in by_name}))
                    return 1e-3, 0.5
                return None

            def close(self):
                pass

        S.install(template_vertices=np.zeros((6890, 3)))
        S.SESSION_FACTORY = Session
        try:
            S.reset(feeds=feeds, params=params, global_step=0)
            with contextlib.redirect_stdout(io.StringIO()):
                from lib import models as RM
                kw = G.reference_kwargs(cfg, h, N, name="fitloop")
                kw["num_epochs"] = 2
                model = holder["model"] = RM.CAPE(**kw)
                model.build_graph(model.input_num_verts, model.nn_input_channel, phase="train")
                model._get_path = lambda folder: os.path.join(tmp, "ref", folder, "fitloop")
                model.evaluate = lambda *a, **k: (ref_log.append(("validate", None)) or ("", 0.25, 0.0, 0.0))
                model.op_saver = types.SimpleNamespace(save=lambda sess, path, global_step=None: ref_log.append(("save", global_step)))
                np.random.seed(11)
                ref_losses, _ = model.fit(data)
        finally:
            S.SESSION_FACTORY = None
    out = {"fit/" + k: v for k, v in fit_stream(ref_log, data).items()}
    out["fit/losses"] = np.asarray(ref_losses, np.float64)
    return out


def ref_predict(G, h):
    from oracle import tf1_shim as S
    N = 2
    data, cond, cond2, labels = predict_inputs()
    with _stubs():
        tag, cfg, _, step = G.configs()[0]
        params, feeds = _shim_feeds(G, cfg, h, N)
        holder = {}

        class Session(object):
            def run(self, fetches, feed_dict=None):
                model = holder["model"]
                x = np.asarray(feed_dict[model.ph_data_g], np.float32)
                c = np.asarray(feed_dict[model.ph_cond_g], np.float32)
                if isinstance(fetches, list):
                    l = predict_losses(x)
                    return predict_out(x, c), l[0], l[1], l[2]
                return predict_out(x, c)

        S.install(template_vertices=np.zeros((6890, 3)))
        S.reset(feeds=feeds, params=params, global_step=0)
        with contextlib.redirect_stdout(io.StringIO()):
            from lib import models as RM
            model = holder["model"] = RM.CAPE(**G.reference_kwargs(cfg, h, N, name="predloop"))
            model.build_graph(model.input_num_verts, model.nn_input_channel, phase="train")
            pred, r, l, e = model.predict(data, cond, cond2, labels, sess=Session())
            string = model.evaluate(data, cond, cond2, labels, sess=Session())
    return {"predict/pred": np.asarray(pred, np.float32).reshape(-1)[::PRED_STRIDE], "predict/pred_shape": np.array(pred.shape),
            "predict/losses": np.array([r, l, e], np.float64), "predict/line": np.array(string[0]),
            "predict/values": np.array(string[1:], np.float64)}


def ref_encode_decode(G, h):
    from oracle import tf1_shim as S
    N = 2
    data, cond, cond2, zt, ye, y2e = encdec_inputs()
    size = data.shape[0]
    with _stubs():
        tag, cfg, _, step = G.configs()[0]
        params, feeds = _shim_feeds(G, cfg, h, N, demo=True)
        holder = {}

        class Session(object):
            def __init__(self, *a, **k):
                pass

            def run(self, fetches, feed_dict=None):
                model = holder["model"]
                fd = {id(k): np.asarray(v, np.float32) for k, v in feed_dict.items() if not isinstance(v, bool)}
                g = lambda ph: fd[id(ph)]
                if not isinstance(fetches, list):
                    return f_dec(g(model.ph_z_total), g(model.ph_y_latent), g(model.ph_y2_latent))
                if len(fetches) == 4:
                    return f_mean(g(model.ph_data_g)), f_var(g(model.ph_data_g)), f_c(g(model.ph_cond_g)), f_c2(g(model.ph_cond2_g))
                return f_c(g(model.ph_cond_g)), f_c2(g(model.ph_cond2_g))

        S.install(template_vertices=np.zeros((6890, 3)))
        S.SESSION_FACTORY = Session
        try:
            S.reset(feeds=feeds, params=params, global_step=0)
            with contextlib.redirect_stdout(io.StringIO()):
                from lib import models as RM
                model = holder["model"] = RM.CAPE(**G.reference_kwargs(cfg, h, N, name="encdec"))
                model.build_graph(model.input_num_verts, model.nn_input_channel, phase="demo")
                enc = model.encode(data, cond, cond2)
                cnd = model.encode_only_condition(cond, cond2)
                dec = model.decode(zt, cond=np.tile(ye, (size, 1)), cond2=np.tile(y2e, (size, 1)))
                dec1 = model.decode(zt, cond=ye, cond2=y2e)                      # one condition row, several codes
        finally:
            S.SESSION_FACTORY = None
    out = {"encdec/enc%d" % i: np.asarray(a) for i, a in enumerate(enc)}
    out.update({"encdec/cond%d" % i: np.asarray(a) for i, a in enumerate(cnd)})
    out["encdec/dec"] = np.asarray(dec, np.float32).reshape(-1)[::PRED_STRIDE]
    out["encdec/dec1"] = np.asarray(dec1, np.float32).reshape(-1)[::PRED_STRIDE]
    out["encdec/dec_shape"] = np.array(dec.shape)
    return out


def ref_lr(G):
    from oracle import tf1_shim as S
    lrs = []
    with _stubs():
        S.install(template_vertices=np.zeros((6890, 3)))
        from lib import models as RM
        for cfg in lr_configs():
            row = []
            for step in LR_STEPS:
                S.reset(params={"generator/w": np.ones(3, np.float32), "discriminator/w": np.ones(3, np.float32)},
                        global_step=step)
                tf = S.tf
                with tf.variable_scope("generator"):
                    wg = tf.get_variable("w", [3])
                with tf.variable_scope("discriminator"):
                    wd = tf.get_variable("w", [3])
                me = types.SimpleNamespace(lr_warmup=cfg["lr_warmup"], optim_condnet=True)
                with contextlib.redirect_stdout(io.StringIO()):
                    RM.CAPE.training(me, loss_g=(wg * wg).sum(), loss_d=(wd * wd).sum(), lr_g=cfg["lr"],
                                     lr_d=cfg["lr"] * cfg["lr_scaler"], optimizer="sgd", decay_steps=cfg["decay_steps"],
                                     decay_rate=cfg["decay_rate"], momentum=0.9)
                S.run_pending()
                assert int(S.GLOBAL_STEP) == step + 2
                row.append(np.asarray(S.RECORD["lr"], np.float64))
            lrs.append(np.stack(row))
    return {"lr/values": np.stack(lrs)}


def ref_flags(G):
    """The add_argument calls of the reference's parse_config, recorded by a stand-in for `configargparse`."""
    recorded = []

    class ArgParser(object):
        def __init__(self, *a, **k):
            pass

        def add_argument(self, flag, **kw):
            recorded.append((flag.lstrip("-"), kw))

        def parse_known_args(self, *a, **k):
            return argparse.Namespace(**{n: kw.get("default") for n, kw in recorded}), []

    stub = types.ModuleType("configargparse")
    stub.ArgParser, stub.ArgumentDefaultsHelpFormatter, stub.DefaultConfigFileParser = ArgParser, object, object
    saved = sys.modules.get("configargparse")
    sys.modules["configargparse"] = stub
    try:
        spec = importlib.util.spec_from_file_location("ref_config_parser", os.path.join(G.REF, "config_parser.py"))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        mod.parse_config()
    finally:
        if saved is None:
            sys.modules.pop("configargparse", None)
        else:
            sys.modules["configargparse"] = saved
    first = recorded[0]
    rest = recorded[1:]
    return {"flags/config": np.array([first[0], repr(bool(first[1].get("is_config_file"))), repr(first[1].get("default"))]),
            "flags/names": np.array([n for n, _ in rest]),
            "flags/types": np.array([kw.get("type", str).__name__ for _, kw in rest]),
            "flags/defaults": np.array([repr(kw.get("default")) for _, kw in rest]),
            "flags/choices": np.array([repr(kw.get("choices")) for _, kw in rest])}


def main():
    import tempfile
    import make_ref_golden as G
    from cape_b200 import topology as T
    if not os.path.isdir(os.path.join(G.REF, "lib")):
        sys.exit("set CAPE_REFERENCE to a checkout of qianlim/CAPE")
    L, D, U, p, L_d, D_d, U_d = T.load_graph_mtx(load_for_demo=True)
    h = dict(L=L, D=D, U=U, p=p, L_d=L_d, D_d=D_d, U_d=U_d)
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        out.update(ref_constructor(G, h))
        os.makedirs(os.path.join(tmp, "body"))
        out.update(ref_body_data(G, os.path.join(tmp, "body")))
        out.update(ref_demo_simple(G, os.path.join(tmp, "demo")))
        out.update(ref_fit(G, h, os.path.join(tmp, "fit")))
    out.update(ref_predict(G, h))
    out.update(ref_encode_decode(G, h))
    out.update(ref_lr(G))
    out.update(ref_flags(G))
    np.savez_compressed(OUT, **out)
    cfg_dir = os.path.join(G.REF, "configs")
    names = sorted(os.listdir(cfg_dir))
    np.savez_compressed(CONFIGS_OUT, names=np.array(names),
                        texts=np.array([open(os.path.join(cfg_dir, n)).read() for n in names]))
    print("wrote", OUT, os.path.getsize(OUT), "bytes;", CONFIGS_OUT, os.path.getsize(CONFIGS_OUT), "bytes")


if __name__ == "__main__":
    sys.path.insert(0, HERE)
    main()
