#!/usr/bin/env python
"""Train-step time of the reference's default model (configs/default_config.yaml: residual encoder blocks, conditioned
encoder, reduce_dim 4, GroupNorm decoder) and where its encoder's time goes.

    python tools/encoder_resblock_step.py OUT_DIR [--batches 16 64] [--steps S] [--warmup W] [--profile-steps R]

For every batch size: one full VAE+GAN update (forward, backward, optimiser) replayed from the two captured CUDA
graphs, timed with CUDA events over S steps after W warm-up steps; then R eager steps with per-launch CUDA events
(engine.PROFILE, as tools/step_profile.py) whose encoder tags (`enc/res3/conv2:fwd`, `...:dx`, `...:dW`, ...) are
reported as per-step medians.  The card name, power limit and SM clock (bench.Clocks, nvidia-smi) go with the
numbers.  Writes OUT_DIR/encoder_resblock_step.json.  Needs a GPU.
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def default_config():
    from cape_b200.params import DEFAULTS
    return dict(DEFAULTS, use_res_block=True, cond_encoder=True, reduce_dim=4, affine=False, lambda_edge=0.0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--batches", type=int, nargs="+", default=[16, 64])
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--profile-steps", type=int, default=5)
    args = ap.parse_args()

    import torch
    assert torch.cuda.is_available(), "encoder_resblock_step.py needs a GPU; there is no CPU fallback"
    import bench
    from cape_b200 import engine as E
    from cape_b200 import topology as T
    from cape_b200.network import CapeNetwork
    from cape_b200.synthetic import make_batch

    cfg = default_config()
    L, D, U, p, L_d, D_d, _ = T.load_graph_mtx(load_for_demo=True)
    torch.cuda.set_device(0)
    clocks = bench.Clocks(0)
    out = {"config": "default_config.yaml (use_res_block 1, cond_encoder 1, reduce_dim 4, affine 0)", "batches": {}}
    for N in args.batches:
        net = CapeNetwork(L, D, U, L_d, D_d, cfg, N, device=0)
        hb = make_batch(N, cfg["nz"], seed=cfg["seed"])
        net.set_inputs(*[torch.from_numpy(hb[k]) for k in ("x_g", "cond_g", "cond2_g", "eps", "x_d", "cond_d", "cond2_d")])
        net.train_step(step=0, update=False)
        torch.cuda.synchronize()
        net.capture_graphs()
        for i in range(args.warmup):
            net.train_step(step=i, use_graph=True)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(args.steps):
            net.train_step(step=args.warmup + i, use_graph=True)
        e1.record()
        torch.cuda.synchronize()
        step_ms = e0.elapsed_time(e1) / args.steps
        per_step = []
        for i in range(args.profile_steps):
            E.PROFILE = []
            net.train_step(step=1000 + i, update=False)
            torch.cuda.synchronize()
            rec = {}
            for family, tag, nbytes, a, b in E.PROFILE:
                if tag.startswith("enc/"):
                    rec[tag] = rec.get(tag, 0.0) + a.elapsed_time(b)
            per_step.append(rec)
        E.PROFILE = None
        tags = sorted({t for r in per_step for t in r})
        layers = {t: statistics.median(r.get(t, 0.0) for r in per_step) for t in tags}
        out["batches"][N] = {"step_ms": step_ms, "meshes_per_s": N / step_ms * 1e3, "encoder_layers_ms": layers,
                             "encoder_ms_sum_eager_profiled": sum(layers.values())}
        print("batch %d: train step %.3f ms (%.1f meshes/s, CUDA graphs, %d steps)" % (N, step_ms, N / step_ms * 1e3,
                                                                                      args.steps))
        for t, ms in sorted(layers.items(), key=lambda kv: -kv[1]):
            print("   %-28s %8.3f ms" % (t, ms))
        del net
        torch.cuda.synchronize()
    out["clocks"] = clocks.stop()
    c = out["clocks"]
    print("%s, power limit %s W, SM clock %s MHz" % (c["gpu"], c["power_limit_w"], c["sm_mhz"]))
    os.makedirs(args.out_dir, exist_ok=True)
    path = os.path.join(args.out_dir, "encoder_resblock_step.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=1)
    print("wrote", path)


if __name__ == "__main__":
    main()
