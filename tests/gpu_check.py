#!/usr/bin/env python
"""Run every parity check on the GPU and print ALL relative errors (no early exit) -- debugging aid;
the pytest -m gpu tests assert on the same functions."""
import json
import os
import sys
import time
import traceback

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))


def truth_table(res):
    """float64-truth mode: print (CUDA error, fp32-oracle error) per tensor, return the part that exceeds the gate
    max(1e-4, 2 x fp32-oracle error) as ratios to it (> 1 fails)."""
    out = {}
    for k, (e, b) in res.items():
        gate = max(1e-4, 2 * b)
        if not k.startswith("param ") and not k.startswith("clipped"):
            print("    %-72s cuda %.2e   fp32-oracle %.2e%s" % (k, e, b, "   <-- over the gate" if e >= gate else ""))
        out[k + " (err / gate)"] = e / gate * 1e-4
    return out


def main():
    import torch
    import parity
    from cape_b200 import topology as T
    from cape_b200.params import NZ64_AFFINE
    L, D, U, p, L_d, D_d, U_d = T.load_graph_mtx(load_for_demo=True)
    h = dict(L=L, D=D, U=U, p=p, L_d=L_d, D_d=D_d)
    cfg = dict(NZ64_AFFINE, decay_steps=10)
    only = sys.argv[1:]
    jobs = [("golden", lambda: parity.golden_ops(h)), ("gemm", parity.gemm_cases),
            ("cheb", lambda: parity.cheb_grad_cases(h)), ("plain", lambda: parity.plain_operand_cases(h)),
            ("plain_fp64", lambda: parity.plain_operand_vs_float64(h)), ("apply", lambda: parity.apply_cases(h)), ("gn", parity.gn_case), ("tc", lambda: parity.tc_vs_simt(h)),
            ("step", lambda: parity.train_step(h, cfg, N=2)),
            ("step_ref", lambda: parity.train_step(h, cfg, N=2, ref_compat=True)),
            ("step_rawinit", lambda: parity.train_step(h, cfg, N=2, fc_scale=1.0)),
            ("step_truth", lambda: truth_table(parity.train_step(h, cfg, N=2, fc_scale=1.0, truth=True))),
            ("step3", lambda: parity.train_step(h, cfg, N=2, nsteps=3, fc_scale=1.0)),
            ("step_n64", lambda: parity.train_step(h, cfg, N=64, use_graph=True, fc_scale=1.0)),
            ("fwd_n32", lambda: parity.generator_forward(h, cfg, N=32)),
            ("step_nomask", lambda: parity.train_step(h, cfg, N=2, impose_masks=False)),
            ("step_n5", lambda: parity.train_step(h, cfg, N=5, seed=7)),
            ("step_gn", lambda: parity.train_step(h, dict(__import__("cape_b200.params", fromlist=["x"]).NZ18_PLAIN,
                                                          decay_steps=10), N=2))]
    allres = {}
    for name, fn in jobs:
        if only and name not in only:
            continue
        t0 = time.time()
        try:
            res = fn()
            torch.cuda.synchronize()
        except Exception:
            traceback.print_exc()
            print("[%s] FAILED" % name)
            continue
        print("[%s] %.1fs" % (name, time.time() - t0))
        for k, v in res.items():
            print("  %-70s %.3e %s" % (k, v, "" if v < parity.TOL else "  <-- FAIL"))
        allres[name] = res
    os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
    json.dump(allres, open(os.path.join(ROOT, "gpurun_out", "gpu_check.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
