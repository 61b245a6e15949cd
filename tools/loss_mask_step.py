#!/usr/bin/env python
"""Cost of `--loss_mask binary`: the affine nz64 train step with and without the mask, and the loss kernel alone.

    python tools/loss_mask_step.py OUT_DIR [--batch 64] [--steps S] [--rounds R] [--warmup W] [--calls C]

Two networks of bench.py's c3 model (affine nz64, L1) at one batch size in one process, one with loss_mask 'binary'.
Each takes full VAE+GAN updates replayed from its two captured CUDA graphs; the two alternate, S steps each per round
over R rounds, timed with CUDA events, and the median over the rounds is reported.  Then C back-to-back calls of the
reconstruction/edge/KL loss (engine.recon_losses: recon_kernel + kl_kernel) on each network's batch, timed the same
way.  The card name, power limit and SM clock (bench.Clocks, nvidia-smi) go with the numbers.  Writes
OUT_DIR/loss_mask_step.json.  Needs a GPU.
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def models():
    from cape_b200.params import NZ64_AFFINE
    return (("affine_nz64", dict(NZ64_AFFINE)), ("affine_nz64_mask", dict(NZ64_AFFINE, loss_mask="binary")))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--calls", type=int, default=200)
    args = ap.parse_args()

    import torch
    assert torch.cuda.is_available(), "loss_mask_step.py needs a GPU; there is no CPU fallback"
    import bench
    from cape_b200 import engine as E
    from cape_b200 import network as NW
    from cape_b200 import topology as T
    from cape_b200.synthetic import make_batch

    L, D, U, p, L_d, D_d, _ = T.load_graph_mtx(load_for_demo=True)
    torch.cuda.set_device(0)
    clocks = bench.Clocks(0)
    N = args.batch
    nets = {}
    for name, cfg in models():
        net = NW.CapeNetwork(L, D, U, L_d, D_d, cfg, N, device=0)
        hb = make_batch(N, cfg["nz"], seed=cfg["seed"])
        net.set_inputs(*[torch.from_numpy(hb[k]) for k in ("x_g", "cond_g", "cond2_g", "eps", "x_d", "cond_d", "cond2_d")])
        net.train_step(step=0, update=False)
        torch.cuda.synchronize()
        net.capture_graphs()
        for i in range(args.warmup):
            net.train_step(step=i, use_graph=True)
        torch.cuda.synchronize()
        nets[name] = net
    assert nets["affine_nz64"].loss_mask is None and nets["affine_nz64_mask"].loss_mask is not None

    def timed(fn, n):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(n):
            fn(i)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n

    times = {name: [] for name in nets}
    for r in range(args.rounds):
        for name, net in nets.items():
            times[name].append(timed(lambda i: net.train_step(step=args.warmup + r * args.steps + i, use_graph=True),
                                     args.steps))

    def loss_call(net, dpred, losses):
        return lambda i: E.recon_losses(net.tp, net.nbr_op, net.x_hat, net.in_x, N, net.p[0], net.recon_kind, 1.0, 1.0,
                                        net.n_edges, net.z_mean, net.z_logvar, net.nz, dpred, losses,
                                        mask=net.loss_mask, mask_sum=net.loss_mask_sum)

    kern = {name: [] for name in nets}
    scratch = {name: (torch.zeros_like(net.d_xhat), torch.zeros(8, device=net.device)) for name, net in nets.items()}
    for name, net in nets.items():
        timed(loss_call(net, *scratch[name]), 20)                             # warm-up
    for r in range(args.rounds):
        for name, net in nets.items():
            kern[name].append(timed(loss_call(net, *scratch[name]), args.calls) * 1e3)

    out = {"batch": N, "steps_per_round": args.steps, "rounds": args.rounds, "loss_calls_per_round": args.calls,
           "models": {}}
    for name in nets:
        step_ms = statistics.median(times[name])
        out["models"][name] = {"step_ms": step_ms, "step_ms_rounds": times[name], "meshes_per_s": N / step_ms * 1e3,
                               "loss_call_us": statistics.median(kern[name]), "loss_call_us_rounds": kern[name]}
        print("%-18s train step %.3f ms median of %d rounds %s (%.1f meshes/s, CUDA graphs, batch %d); loss call "
              "%.2f us %s" % (name, step_ms, args.rounds, ["%.3f" % t for t in times[name]], N / step_ms * 1e3, N,
                              statistics.median(kern[name]), ["%.2f" % t for t in kern[name]]))
    out["clocks"] = clocks.stop()
    c = out["clocks"]
    print("%s, power limit %s W, SM clock %s MHz" % (c["gpu"], c["power_limit_w"], c["sm_mhz"]))
    os.makedirs(args.out_dir, exist_ok=True)
    path = os.path.join(args.out_dir, "loss_mask_step.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=1)
    print("wrote", path)


if __name__ == "__main__":
    main()
