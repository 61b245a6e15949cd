#!/usr/bin/env python
"""What each column tile of a fused conv launch costs: one conv_wg_kernel launch at the `enc/conv8` forward shape of the
c3 network, timed at ncols = 128, 256 and 512.

    python tools/conv_tile_cost.py OUT_DIR [--launches L] [--windows W]

Builds the c3 CapeNetwork as bench.py does, runs one generator forward to record the arguments of the layer's fused
`cheb_call` (rows, terms, operators, condition, epilogue), then launches that call alone with only the first ncols
output columns (the same weights, biases and condition weights, sliced).  Every launch gathers the same basis chunks;
only the column tiles differ.  A second case contracts the same shape with plain operands (every term an identity
operator, the plain-operand launcher) for comparison.  For each case and ncols: median over W windows of the mean
launch time over L back-to-back launches (CUDA events), and the time per 128 output columns.  The card name, power
limit and SM clock (bench.Clocks) go with the numbers.  Writes OUT_DIR/conv_tile_cost.json and prints a table.  Needs
a GPU.
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

TAG = "enc/conv8:fwd"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--launches", type=int, default=50, help="back-to-back launches per timed window")
    ap.add_argument("--windows", type=int, default=7)
    args = ap.parse_args()

    import torch
    assert torch.cuda.is_available(), "conv_tile_cost.py needs a GPU; there is no CPU fallback"
    import bench
    from cape_b200 import engine as E
    from cape_b200 import network as NW
    from cape_b200.network import CapeNetwork
    from cape_b200.synthetic import make_batch

    cfg, h = bench.config_and_hierarchy("c3")
    N = bench.CONFIGS["c3"]["batch"]
    torch.cuda.set_device(0)
    net = CapeNetwork(h["L"], h["D"], h["U"], h["L_d"], h["D_d"], cfg, N, device=0)
    net.prep_weights()
    hb = make_batch(N, cfg["nz"], seed=cfg["seed"])
    net.set_inputs(*[torch.from_numpy(hb[k]) for k in ("x_g", "cond_g", "cond2_g", "eps", "x_d", "cond_d", "cond2_d")])

    seen = []
    cheb_call = NW.cheb_call

    def record(tp, n, rows_out, ncols, terms, out, **k):
        if k.get("tag") is not None and k["tag"][0] == TAG:
            seen.append((tp, n, rows_out, ncols, [dict(t) for t in terms], k))
        return cheb_call(tp, n, rows_out, ncols, terms, out, **k)

    NW.cheb_call = record
    net.forward_generator()
    torch.cuda.synchronize()
    NW.cheb_call = cheb_call
    assert seen, "the forward made no fused call tagged " + TAG
    tp, n, rows_out, full_cols, terms, kw = seen[0]
    kw = {k: v for k, v in kw.items() if k != "tag"}
    assert full_cols >= 512 and kw.get("out2") is None

    # the same contraction with plain operands: each term's basis as its own [N, rows_out, F] tensor
    g = torch.Generator(device="cuda").manual_seed(0)
    plain = []
    for t in terms:
        src = torch.randn(n, rows_out, t["F"], device="cuda", generator=g)
        plain.append(dict(t, src=src, op=-1, src_rows=rows_out, src_stride=t["F"], stash=None, stash_stride=0))
    plain_kw = dict(kw, cond=None)

    def time_call(case_terms, case_kw, ncols):
        out = torch.empty(n, rows_out, ncols, device="cuda")
        for _ in range(3):
            E.cheb_call(tp, n, rows_out, ncols, case_terms, out, **case_kw)
        torch.cuda.synchronize()
        per = []
        for _ in range(args.windows):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.launches):
                E.cheb_call(tp, n, rows_out, ncols, case_terms, out, **case_kw)
            e1.record()
            e1.synchronize()
            per.append(e0.elapsed_time(e1) / args.launches)
        return statistics.median(per), (max(per) - min(per)) / 2

    clocks = bench.Clocks(0)
    rows = []
    for case, case_terms, case_kw in (("fused", terms, kw), ("plain", plain, plain_kw)):
        for ncols in (128, 256, 512):
            ms, spread = time_call(case_terms, case_kw, ncols)
            rows.append({"case": case, "ncols": ncols, "ms": ms, "spread_ms": spread, "ms_per_128_cols": ms * 128 / ncols})
    clk = clocks.stop()

    result = {"layer": TAG, "N": n, "rows_out": rows_out, "terms": [(t["op"], t["F"]) for t in terms],
              "slots": sum(1 for t in terms if t.get("wc") is not None), "clocks": clk, "launches": rows}
    os.makedirs(args.out_dir, exist_ok=True)
    path = os.path.join(args.out_dir, "conv_tile_cost.json")
    with open(path, "w") as f:
        json.dump(result, f, indent=1)
    print("%s: N %d, rows_out %d, terms %s; %s, %s W, SM %s MHz"
          % (TAG, n, rows_out, result["terms"], clk["gpu"], clk["power_limit_w"], clk["sm_mhz"]))
    print("%-6s %6s %9s %9s %12s" % ("case", "ncols", "ms", "+-", "ms/128 cols"))
    for r in rows:
        print("%-6s %6d %9.4f %9.4f %12.4f" % (r["case"], r["ncols"], r["ms"], r["spread_ms"], r["ms_per_128_cols"]))
    print("wrote", path)


if __name__ == "__main__":
    main()
