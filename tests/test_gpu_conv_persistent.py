"""The persistent tile loop of the wgmma convolution kernel (conv_wg_kernel): launches with several times more tiles
than the H100 has SMs, so that each CTA takes several tiles and different CTAs take different numbers of them, and the
ring's stage and phase cross tile boundaries at every offset.  The loop runs at BN = 32 and 64 (ncols <= 64, and
ncols <= 32 with two accumulators); the wider and the dual BN = 64 instantiations run one tile per CTA and are covered
at the same sizes.  Checked against a float64 NumPy product by the harness of test_gpu_conv_ring.py.  The last case
replays one launch from a captured CUDA graph and eagerly: the tile counter of the topology handle must be back at
zero after every launch."""
import numpy as np
import pytest
import torch

from test_gpu_conv_ring import _operator, run_case

pytestmark = pytest.mark.gpu


# 1, 2, 5 and 14 chunks per tile; 128-row tiles: 394 to 782 tiles over 132 SMs.  One chunk is only reachable through
# the plain-operand contraction (a 32-deep reduction).
@pytest.mark.parametrize("N,M,ncols,Fs,gather", [
    (40, 2000, 64, [32], [False]),
    (24, 2100, 64, [64], [True]),
    (20, 2500, 48, [96, 64], [False, False]),   # plain operands: a partial column tile of 48 in a BN = 64 tile
    (20, 2500, 160, [96, 64], [True, False]),   # one tile per CTA: two column tiles, the last one partial
    (10, 6000, 64, [224, 224], [True, True]),
])
def test_many_tiles(N, M, ncols, Fs, gather):
    run_case(N=N, M=M, ncols=ncols, Fs=Fs, gather=gather)


# rows_out = 203: consecutive tiles of one CTA cover different samples, so the condition vectors are refreshed per tile
@pytest.mark.parametrize("ncols", [32, 160])
def test_many_tiles_condition_slots(ncols):
    run_case(N=300, M=203, ncols=ncols, Fs=[64, 48], gather=[True, False], slots=2)


# the dual-accumulator affine epilogue with the basis stash, written by the first column tile of each row tile
@pytest.mark.parametrize("ncols", [32, 64])
def test_many_tiles_affine_dual_with_stash(ncols):
    run_case(N=30, M=2000, ncols=ncols, Fs=[96, 96], gather=[False, True], dual=True, slots=1, epilogue="affine",
             stash=True)


@pytest.mark.parametrize("ncols", [64, 160])
@pytest.mark.parametrize("epilogue", ["slope", "dualmask"])
def test_many_tiles_data_gradient_epilogues(epilogue, ncols):
    run_case(N=25, M=2111, ncols=ncols, Fs=[128, 128], gather=[True, True], epilogue=epilogue)


# pass-through terms (the encoder's residual skip): an identity and a gathered one, added in the epilogue
def test_many_tiles_pass_through():
    from cape_b200 import engine as E
    from cape_b200 import ops
    dev = torch.device("cuda", 0)
    tp = ops.topology_for(dev)
    rng = np.random.RandomState(3)
    N, M, F, ncols = 24, 2100, 96, 64
    src = rng.normal(size=(N, M, F)).astype(np.float32)
    m = _operator(rng, M)
    op = tp.add_operator(m)
    w = rng.normal(0, 1 / np.sqrt(F), size=(F, ncols)).astype(np.float32)
    skip = rng.normal(size=(N, M, ncols)).astype(np.float32)
    ms = _operator(rng, M)
    ops_ = tp.add_operator(ms)
    skip2 = rng.normal(size=(N, M, ncols)).astype(np.float32)
    t = lambda a: torch.from_numpy(a).to(dev)
    terms = [dict(src=t(src), op=op, F=F, src_rows=M, src_stride=F, w=t(w), w_stride=ncols, wT=t(w.T.copy()),
                  wT_stride=F),
             dict(src=t(skip), op=-1, F=ncols, src_rows=M, src_stride=ncols, w_stride=0),
             dict(src=t(skip2), op=ops_, F=ncols, src_rows=M, src_stride=ncols, w_stride=0)]
    out = torch.empty(N, M, ncols, device=dev)
    E.cheb_call(tp, N, M, ncols, terms, out)
    torch.cuda.synchronize()
    m64, ms64 = m.astype(np.float64), ms.astype(np.float64)
    want = np.stack([m64 @ src[n].astype(np.float64) @ w.astype(np.float64) + skip[n] + ms64 @ skip2[n]
                     for n in range(N)])
    got = out.cpu().numpy()
    assert np.abs(got - want).max() / np.abs(want).max() < 1e-4


# one launch three times from a captured graph, and twice eagerly: every run draws its tiles from a counter at zero
def test_graph_replay_and_eager_launches_agree():
    from cape_b200 import engine as E
    from cape_b200 import ops
    dev = torch.device("cuda", 0)
    tp = ops.topology_for(dev)
    rng = np.random.RandomState(7)
    N, M, F, ncols = 20, 2500, 96, 64
    m = _operator(rng, M)
    op = tp.add_operator(m)
    t = lambda a: torch.from_numpy(a).to(dev)
    src = rng.normal(size=(N, M, F)).astype(np.float32)
    w = rng.normal(0, 1 / np.sqrt(F), size=(F, ncols)).astype(np.float32)
    terms = [dict(src=t(src), op=op, F=F, src_rows=M, src_stride=F, w=t(w), w_stride=ncols, wT=t(w.T.copy()),
                  wT_stride=F)]
    s = torch.cuda.Stream(device=dev)
    s.wait_stream(torch.cuda.current_stream())
    outs = []
    with torch.cuda.stream(s):
        out = torch.full((N, M, ncols), float("nan"), device=dev)
        E.cheb_call(tp, N, M, ncols, terms, out)
        outs.append(out.clone())
        g = torch.cuda.CUDAGraph()
        gout = torch.full((N, M, ncols), float("nan"), device=dev)
        with torch.cuda.graph(g, stream=s):
            E.cheb_call(tp, N, M, ncols, terms, gout)
        for _ in range(3):
            gout.fill_(float("nan"))
            g.replay()
            outs.append(gout.clone())
        out.fill_(float("nan"))
        E.cheb_call(tp, N, M, ncols, terms, out)
        outs.append(out.clone())
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    want = np.stack([m.astype(np.float64) @ src[n].astype(np.float64) @ w.astype(np.float64) for n in range(N)])
    first = outs[0].cpu().numpy()
    assert np.abs(first - want).max() / np.abs(want).max() < 1e-4
    for o in outs[1:]:
        assert np.array_equal(o.cpu().numpy(), first)
