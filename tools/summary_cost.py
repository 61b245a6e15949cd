#!/usr/bin/env python
"""Cost of `CAPE(summary_dir=...)`: the summary point of fit and the per-application moving average, next to the eager
training step that fit runs.

    python tools/summary_cost.py OUT_DIR [--batch 64] [--steps S] [--rounds R] [--warmup W] [--points P]

For affine nz64 and GroupNorm nz18 at one batch size, in one process:
  * the eager update of fit (CapeNetwork.train_step, no CUDA graphs), without and with the moving average (one
    cape_sumsq per regularised FC kernel + cape_loss_ema between the backward pass and the update), alternating, S steps
    per round over R rounds, CUDA events, median over the rounds;
  * the summary point, host clock around work that ends in a synchronise, P points per round: the forward pass
    (enqueue_loss_forward), cape_histogram and its device-to-host copy (weight_histograms), and encoding plus
    writing one event (CAPE._summary_values + EventWriter.add, the whole point as fit runs it), each reported apart.
The card name, power limit and SM clock (bench.Clocks, nvidia-smi) go with the numbers.  Writes
OUT_DIR/summary_cost.json.  Needs a GPU.
"""
import argparse
import gc
import json
import os
import statistics
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def models():
    from cape_b200.params import NZ18_PLAIN, NZ64_AFFINE
    return (("affine_nz64", dict(NZ64_AFFINE)), ("groupnorm_nz18", dict(NZ18_PLAIN)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--points", type=int, default=5)
    args = ap.parse_args()

    import torch
    assert torch.cuda.is_available(), "summary_cost.py needs a GPU; there is no CPU fallback"
    import bench
    from cape_b200 import topology as T
    from cape_b200.models import CAPE
    from cape_b200.synthetic import make_batch

    L, D, U, p, L_d, D_d, _ = T.load_graph_mtx(load_for_demo=True)
    torch.cuda.set_device(0)
    clocks = bench.Clocks(0)
    N = args.batch
    out = {"batch": N, "steps_per_round": args.steps, "rounds": args.rounds, "points_per_round": args.points,
           "models": {}}
    tmp = tempfile.mkdtemp(prefix="summary_cost_")

    def timed(fn, n):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(n):
            fn(i)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n

    def host(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3

    for name, cfg in models():
        kw = {k: cfg[k] for k in ("F", "K", "Kd", "nz", "nz_cond", "nz_cond2", "cond_dim", "cond2_dim", "affine",
                                  "use_res_block", "use_res_block_dec", "cond_encoder", "lr_warmup", "regularization",
                                  "lambda_gan", "lr_scaler")}
        m = CAPE(L=L, D=D, U=U, L_d=L_d, D_d=D_d, p=p, batch_size=N, summary_dir=tmp, name=name, restart=True, **kw)
        m.build_graph(m.input_num_verts, m.nn_input_channel)
        net = m.net
        hb = make_batch(N, cfg["nz"], seed=cfg["seed"])
        net.set_inputs(*[torch.from_numpy(hb[k]) for k in ("x_g", "cond_g", "cond2_g", "eps", "x_d", "cond_d", "cond2_d")])
        writer = m._open_summaries()                      # also switches the moving average on
        avg = net.loss_avg
        step = 0

        def train(with_avg):
            def fn(i):
                nonlocal step
                net.loss_avg = avg if with_avg else None
                net.train_step(step=step)
                step += 1
            return fn

        for w in (False, True):
            timed(train(w), args.warmup)
        eager = {False: [], True: []}
        for r in range(args.rounds):
            for w in (False, True):
                eager[w].append(timed(train(w), args.steps))
        net.loss_avg = avg
        ema = []
        timed(lambda i: net.enqueue_loss_average(), 20)
        for r in range(args.rounds):
            ema.append(timed(lambda i: net.enqueue_loss_average(), 200) * 1e3)

        parts = {"forward": [], "histogram": [], "point": []}
        for r in range(args.rounds + 1):                  # round 0 warms up (lazy histogram buffers)
            fw = statistics.median(host(lambda: net.enqueue_loss_forward()) for _ in range(args.points))
            hi = statistics.median(host(lambda: net.weight_histograms()) for _ in range(args.points))
            pt = statistics.median(host(lambda: writer.add(step, *m._summary_values())) for _ in range(args.points))
            if r:
                parts["forward"].append(fw)
                parts["histogram"].append(hi)
                parts["point"].append(pt)
        writer.close()
        res = {"eager_step_ms": statistics.median(eager[False]), "eager_step_ms_rounds": eager[False],
               "eager_step_with_average_ms": statistics.median(eager[True]),
               "eager_step_with_average_ms_rounds": eager[True],
               "sumsq_plus_ema_us": statistics.median(ema), "sumsq_plus_ema_us_rounds": ema}
        for k, v in parts.items():
            res[k + "_ms"] = statistics.median(v)
            res[k + "_ms_rounds"] = v
        res["event_bytes"] = os.path.getsize(writer.path)
        out["models"][name] = res
        print("%-15s eager step %.3f ms, with the moving average %.3f ms; cape_sumsq x3 + cape_loss_ema %.1f us alone"
              % (name, res["eager_step_ms"], res["eager_step_with_average_ms"], res["sumsq_plus_ema_us"]))
        print("%-15s summary point %.2f ms (forward %.2f ms, cape_histogram + copy %.2f ms; the rest is encoding and "
              "writing), batch %d" % (name, res["point_ms"], res["forward_ms"], res["histogram_ms"], N))
        del m, net, writer
        gc.collect()
        torch.cuda.empty_cache()
    out["clocks"] = clocks.stop()
    c = out["clocks"]
    print("%s, power limit %s W, SM clock %s MHz" % (c["gpu"], c["power_limit_w"], c["sm_mhz"]))
    os.makedirs(args.out_dir, exist_ok=True)
    path = os.path.join(args.out_dir, "summary_cost.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=1)
    print("wrote", path)


if __name__ == "__main__":
    main()
