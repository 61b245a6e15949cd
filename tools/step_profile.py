#!/usr/bin/env python
"""Per-layer profile of one bench.py workload: where the step's time goes, set against the H100's two bounds.

    python tools/step_profile.py OUT_DIR [--config c3|c2|c5] [--steps R] [--warmup W]

Builds the CapeNetwork of the config exactly as bench.py does, warms up, then runs R eager steps with per-launch CUDA
events (engine.PROFILE, as bench.py's roofline pass).  Records are grouped by tag (`enc/conv8:fwd`, `...:dx`, `...:dW`,
...); for each tag the per-step sum of its launches is taken and the median over the R steps is reported with:
  - launches per step,
  - the algorithmic bytes the layer books (ChebLayer.alg_bytes) and the achieved GB/s,
  - the contraction FLOPs from the call's shapes (rows x Kred x Fout x 2, x3 for the 3xTF32 passes) and TFLOP/s,
  - which bound is larger (HBM at 3.35 TB/s or TF32 tensor at 495 TFLOP/s, H100 SXM data sheet) and the tag's
    share of that bound (bound time / measured time),
  - the tag's share of the profiled step.
The card name, power limit and SM clock, sampled with nvidia-smi over the profiled steps (bench.Clocks), go with the
table.  Per-launch events slow an eager step: use this to rank layers and bench.py for step times.  Writes
OUT_DIR/step_profile_<config>.json and prints the table.  Needs a GPU.
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BPS = 3.35e12        # H100 SXM data sheet, HBM3
TF32_FLOPS = 495e12      # H100 SXM data sheet, dense TF32 tensor
TF32_PASSES = 3          # 3xTF32: a_hi*b_hi + a_lo*b_hi + a_hi*b_lo


def _contraction_counter(E, modules):
    """Wraps the engine's contraction helpers so every tagged call adds its FLOPs (1x count) to `flops[tag]`."""
    flops = {}

    def add(tag, n):
        if E.PROFILE is not None and tag is not None:
            flops[tag[0]] = flops.get(tag[0], 0.0) + float(n)

    cheb_call, cheb_dw, gemm = E.cheb_call, E.cheb_dw, E.gemm

    def cheb_call_counted(tp, N, rows_out, ncols, terms, *a, **k):
        dual = any(t.get("w2") is not None for t in terms)
        add(k.get("tag"), 2.0 * N * rows_out * ncols * sum(t["F"] for t in terms) * (2 if dual else 1))
        return cheb_call(tp, N, rows_out, ncols, terms, *a, **k)

    def cheb_dw_counted(tp, N, rows_out, ncols, src, op, F, *a, **k):
        nops = len(op) if isinstance(op, (list, tuple)) else 1
        add(k.get("tag"), 2.0 * N * rows_out * ncols * F * nops)
        return cheb_dw(tp, N, rows_out, ncols, src, op, F, *a, **k)

    def gemm_counted(tp, A, B, Cout, *a, **k):
        add(k.get("tag"), 2.0 * A.shape[0] * A.shape[1] * B.shape[1])
        return gemm(tp, A, B, Cout, *a, **k)

    for m in modules:
        for name, fn in (("cheb_call", cheb_call_counted), ("cheb_dw", cheb_dw_counted), ("gemm", gemm_counted)):
            if hasattr(m, name):
                setattr(m, name, fn)
    return flops


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--config", default="c3", choices=["c2", "c3", "c5"])
    ap.add_argument("--steps", type=int, default=7, help="profiled steps (>= 5)")
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    assert args.steps >= 5, "--steps must be >= 5"

    import torch
    assert torch.cuda.is_available(), "step_profile.py needs a GPU; there is no CPU fallback"
    import bench
    from cape_b200 import engine as E
    from cape_b200 import network as NW
    from cape_b200.network import CapeNetwork
    from cape_b200.synthetic import make_batch

    c = bench.CONFIGS[args.config]
    train = c["mode"] == "train"
    cfg, h = bench.config_and_hierarchy(args.config)
    N = c["batch"]
    torch.cuda.set_device(0)
    net = CapeNetwork(h["L"], h["D"], h["U"], h["L_d"], h["D_d"], cfg, N, device=0)
    net.prep_weights()
    hb = make_batch(N, cfg["nz"], seed=cfg["seed"])
    order = ("x_g", "cond_g", "cond2_g", "eps", "x_d", "cond_d", "cond2_d") if train else ("x_g", "cond_g", "cond2_g", "eps")
    net.set_inputs(*[torch.from_numpy(hb[k]) for k in order])
    flops = _contraction_counter(E, [E, NW])

    def step(i):
        if train:
            net.train_step(step=i, allreduce=None, update=False)
        else:
            net.forward_generator()

    clocks = bench.Clocks(0)    # started before the warm-up: nvidia-smi needs a moment before its first sample
    for i in range(args.warmup):
        step(500 + i)
    torch.cuda.synchronize()

    per_step = []           # [{tag: [ms, launches, bytes, flops]}]
    for i in range(args.steps):
        E.PROFILE = []
        flops.clear()
        step(600 + i)
        torch.cuda.synchronize()
        rec = {}
        for family, tag, nbytes, e0, e1 in E.PROFILE:
            r = rec.setdefault(tag, [0.0, 0, 0.0, 0.0, family])
            r[0] += e0.elapsed_time(e1)
            r[1] += 1
            r[2] += nbytes
        for tag, f in flops.items():
            rec.setdefault(tag, [0.0, 0, 0.0, 0.0, "?"])[3] = f
        per_step.append(rec)
    E.PROFILE = None
    clk = clocks.stop()

    tags = sorted({t for r in per_step for t in r})
    rows = []
    for tag in tags:
        ms = statistics.median(r[tag][0] if tag in r else 0.0 for r in per_step)
        last = next(r[tag] for r in reversed(per_step) if tag in r)
        _, launches, nbytes, fl, family = last
        t_hbm = nbytes / HBM_BPS * 1e3
        t_tc = fl * TF32_PASSES / TF32_FLOPS * 1e3
        bound_ms = max(t_hbm, t_tc)
        rows.append({"tag": tag, "family": family, "ms": ms, "launches": launches, "alg_bytes": nbytes,
                     "GBps": nbytes / (ms * 1e-3) / 1e9 if ms > 0 else None, "flops_1x": fl,
                     "TFLOPs_3xtf32": fl * TF32_PASSES / (ms * 1e-3) / 1e12 if ms > 0 else None,
                     "bound": "tensor" if t_tc > t_hbm else "hbm", "bound_ms": bound_ms,
                     "share_of_bound": bound_ms / ms if ms > 0 else None})
    total = sum(r["ms"] for r in rows)
    for r in rows:
        r["share_of_step"] = r["ms"] / total if total > 0 else None
    rows.sort(key=lambda r: -r["ms"])
    result = {"config": args.config, "batch": N, "profiled_steps": args.steps, "profiled_step_ms": total,
              "bound_ms_sum": sum(r["bound_ms"] for r in rows), "clocks": clk,
              "peaks": {"hbm_GBps": HBM_BPS / 1e9, "tf32_TFLOPs": TF32_FLOPS / 1e12, "source": "H100 SXM data sheet"},
              "tags": rows}
    os.makedirs(args.out_dir, exist_ok=True)
    path = os.path.join(args.out_dir, "step_profile_%s.json" % args.config)
    with open(path, "w") as f:
        json.dump(result, f, indent=1)

    print("%s batch %d: profiled step %.2f ms (sum of tag medians), bounds sum %.2f ms; %s, %s W, SM %s MHz"
          % (args.config, N, total, result["bound_ms_sum"], clk["gpu"], clk["power_limit_w"], clk["sm_mhz"]))
    print("%-28s %8s %5s %8s %8s %8s %6s %7s %6s" % ("tag", "ms", "n", "GB", "GB/s", "TFLOP/s", "bound", "of bnd",
                                                      "step"))
    for r in rows:
        print("%-28s %8.3f %5d %8.3f %8.1f %8.1f %6s %6.1f%% %5.1f%%"
              % (r["tag"][:28], r["ms"], r["launches"], r["alg_bytes"] / 1e9, r["GBps"] or 0.0,
                 r["TFLOPs_3xtf32"] or 0.0, r["bound"], 100 * (r["share_of_bound"] or 0.0),
                 100 * (r["share_of_step"] or 0.0)))
    print("wrote", path)


if __name__ == "__main__":
    main()
