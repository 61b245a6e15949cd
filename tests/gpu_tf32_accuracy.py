#!/usr/bin/env python
"""Debug runner: accuracy of the 3xTF32 tensor-core contraction against a float64 truth, per layer shape, next to the
fp32 SIMT kernel.  Prints max-abs/max-ref and rms relative errors of the forward output."""
import os
import sys

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def main():
    import numpy as np
    import torch
    import parity
    from oracle import cape_oracle as O
    from cape_b200 import _lib, ops
    from cape_b200 import topology as T
    lib = _lib.load()
    L, D, U, p, L_d, D_d, U_d = T.load_graph_mtx(load_for_demo=True)
    o = O.Oracle(L, D, U, L_d, D_d, dict(F=[64] * 8, K=[2] * 8, Kd=3), dtype=torch.float64)
    g = torch.Generator(device="cuda").manual_seed(1)
    cases = [("L1 64->64 K=2", 1, 2, 64, 64, 4), ("L3 128->128 K=2", 3, 2, 128, 128, 4),
             ("L5 256->256 K=2", 5, 2, 256, 256, 4), ("L7 512->512 K=2", 7, 2, 512, 512, 8),
             ("L7 512->64 K=1", 7, 1, 512, 64, 8)]
    for tag, lvl, K, Fin, Fout, N in cases:
        x = torch.randn(N, L[lvl].shape[0], Fin, device="cuda", generator=g)
        x = torch.where(x > 0, x, 0.2 * x)                       # like a leaky-ReLU output: non-zero mean
        W = torch.randn(Fin * K, Fout, device="cuda", generator=g) * 0.1
        want = o.chebyshev5(x.cpu().double(), o.Lt[lvl], W.cpu().double(), K).numpy()
        res = {}
        for name, tc in (("simt", 0), ("tensor cores", 1)):
            prev = lib.cape_set_tensor_cores(tc)
            y = ops.chebyshev5(x, L[lvl], W, K).cpu().numpy().astype(np.float64)
            lib.cape_set_tensor_cores(prev)
            e = y - want
            res[name] = (np.abs(e).max() / np.abs(want).max(), np.sqrt((e ** 2).mean() / (want ** 2).mean()),
                         e.mean() / np.abs(want).mean(), (e * np.sign(want)).mean() / np.abs(want).mean())
        print(tag)
        for k, v in res.items():
            print("   %-28s max-rel %.2e   rms-rel %.2e   mean(e)/mean|y| %+.2e   mean(e*sign y)/mean|y| %+.2e" % ((k,) + v))


if __name__ == "__main__":
    main()
