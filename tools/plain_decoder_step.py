#!/usr/bin/env python
"""Train-step time of the plain decoder (`--use_res_block_dec 0`) and of `--reduce_dim 0`, next to the benchmarked
affine nz64 model, and where their decoder and FC time goes.

    python tools/plain_decoder_step.py OUT_DIR [--batch 64] [--steps S] [--rounds R] [--warmup W] [--profile-steps P]

Four models at one batch size, all built in one process: affine nz64 (bench.py's c3, the anchor), plain nz18, plain
nz64, and plain nz64 with reduce_dim 0.  Each takes full VAE+GAN updates (forward, backward, optimiser) replayed from its
two captured CUDA graphs; the models alternate, S steps each per round over R rounds, timed with CUDA events, and the
median over the rounds is reported.  Then P eager steps per model with per-launch CUDA events (engine.PROFILE, as
tools/step_profile.py): the per-step medians of the `dec/conv*` tags, and of the FC layers (their forward tags, and CUDA
events around each FC layer's backward call).  The card name, power limit and SM clock (bench.Clocks, nvidia-smi) go
with the numbers.  Writes OUT_DIR/plain_decoder_step.json.  Needs a GPU.
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def models():
    from cape_b200.params import NZ18_PLAIN, NZ64_AFFINE
    return (("affine_nz64", dict(NZ64_AFFINE)),
            ("plain_nz18", dict(NZ18_PLAIN, use_res_block_dec=False)),
            ("plain_nz64", dict(NZ64_AFFINE, use_res_block_dec=False)),
            ("plain_nz64_rd0", dict(NZ64_AFFINE, use_res_block_dec=False, reduce_dim=0)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--profile-steps", type=int, default=5)
    args = ap.parse_args()

    import torch
    assert torch.cuda.is_available(), "plain_decoder_step.py needs a GPU; there is no CPU fallback"
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
    times = {name: [] for name in nets}
    for r in range(args.rounds):
        for name, net in nets.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for i in range(args.steps):
                net.train_step(step=args.warmup + r * args.steps + i, use_graph=True)
            e1.record()
            torch.cuda.synchronize()
            times[name].append(e0.elapsed_time(e1) / args.steps)

    # FC backward calls are not tagged launches: CUDA events around each call of Dense.bwd while profiling
    dense_bwd = NW.Dense.bwd

    def timed_bwd(self, *a, **kw):
        if E.PROFILE is None or not self.name.startswith(("encoder/", "decoder/")):
            return dense_bwd(self, *a, **kw)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        dense_bwd(self, *a, **kw)
        e1.record()
        E.PROFILE.append(("dense_bwd", self.name + ":bwd", 0, e0, e1))

    NW.Dense.bwd = timed_bwd
    out = {"batch": N, "steps_per_round": args.steps, "rounds": args.rounds, "models": {}}
    try:
        for name, net in nets.items():
            per_step = []
            for i in range(args.profile_steps):
                E.PROFILE = []
                net.train_step(step=1000 + i, update=False)
                torch.cuda.synchronize()
                rec = {}
                for family, tag, nbytes, a, b in E.PROFILE:
                    if tag.startswith(("dec/conv", "encoder/fc", "decoder/fc")):
                        rec[tag] = rec.get(tag, 0.0) + a.elapsed_time(b)
                per_step.append(rec)
            E.PROFILE = None
            tags = sorted({t for r in per_step for t in r})
            layers = {t: statistics.median(r.get(t, 0.0) for r in per_step) for t in tags}
            step_ms = statistics.median(times[name])
            out["models"][name] = {"step_ms": step_ms, "step_ms_rounds": times[name], "meshes_per_s": N / step_ms * 1e3,
                                   "layers_ms_eager_profiled": layers}
            print("%-16s train step %.3f ms median of %d rounds %s (%.1f meshes/s, CUDA graphs, batch %d)"
                  % (name, step_ms, args.rounds, ["%.3f" % t for t in times[name]], N / step_ms * 1e3, N))
            for t, ms in sorted(layers.items(), key=lambda kv: -kv[1]):
                print("   %-28s %8.3f ms" % (t, ms))
    finally:
        NW.Dense.bwd = dense_bwd
        E.PROFILE = None
    out["clocks"] = clocks.stop()
    c = out["clocks"]
    print("%s, power limit %s W, SM clock %s MHz" % (c["gpu"], c["power_limit_w"], c["sm_mhz"]))
    os.makedirs(args.out_dir, exist_ok=True)
    path = os.path.join(args.out_dir, "plain_decoder_step.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=1)
    print("wrote", path)


if __name__ == "__main__":
    main()
