"""The weight tiles of the wgmma convolution kernel (conv_wg_kernel) arrive by TMA from the terms' K-major weight copies,
and every instantiation runs the persistent tile loop.  Launches with several tiles per CTA at BN = 128 and at BN = 64
with two accumulators; weights given as strided views (the Wt[:, k, :] slices of ops.py), reductions whose F is not a
multiple of 32 (the zero-filled end of the k box), column counts that end part-way through a column tile (the
zero-filled end of the column box), and a two-accumulator call in which one term has no second weight.  Checked
against float64 NumPy products."""
import numpy as np
import pytest
import torch

from test_gpu_conv_ring import _operator, _rel, run_case

pytestmark = pytest.mark.gpu

TOL = 1e-4


# BN = 128: 394 to 1576 tiles over 132 SMs; 160 and 480 end part-way through their last column tile
@pytest.mark.parametrize("ncols", [160, 256, 480, 512])
def test_many_wide_tiles(ncols):
    run_case(N=20, M=2500, ncols=ncols, Fs=[96, 64], gather=[True, False])


# F % 32 != 0 in every term: each term's last chunk reads past F, which the box fills with zeros
def test_many_wide_tiles_partial_chunks():
    run_case(N=10, M=5000, ncols=256, Fs=[40, 72, 100], gather=[True, False, True])


# two accumulators at BN = 64, with condition slots on both and the basis stash
@pytest.mark.parametrize("ncols", [128, 256])
def test_many_tiles_affine_dual_wide(ncols):
    run_case(N=30, M=2000, ncols=ncols, Fs=[96, 72], gather=[False, True], dual=True, slots=1, epilogue="affine",
             stash=True)


@pytest.mark.parametrize("epilogue", ["slope", "dualmask"])
def test_many_wide_tiles_data_gradient_epilogues(epilogue):
    run_case(N=25, M=2111, ncols=288, Fs=[128, 128], gather=[True, True], epilogue=epilogue)


def _ctx():
    from cape_b200 import engine as E
    from cape_b200 import ops
    dev = torch.device("cuda", 0)
    return E, ops.topology_for(dev), dev


# the weights of each term a [ncols, F] slice of one [ncols, K, F] tensor: row stride K * F, offset k * F
@pytest.mark.parametrize("dual,ncols", [(False, 256), (False, 160), (True, 128)])
def test_strided_weight_views(dual, ncols):
    E, tp, dev = _ctx()
    rng = np.random.RandomState(11 + ncols)
    N, M, F, K = 12, 2300, 72, 3
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    Wt = rng.normal(0, 1 / np.sqrt(F), size=(ncols, K, F)).astype(np.float32)
    Wt2 = rng.normal(0, 1 / np.sqrt(F), size=(ncols, K, F)).astype(np.float32)
    Wt_d, Wt2_d = t(Wt), t(Wt2)
    v0 = np.zeros((N, M, ncols))
    v1 = np.zeros((N, M, ncols))
    terms = []
    for k in range(K):
        src = rng.normal(size=(N, M, F)).astype(np.float32)
        m = _operator(rng, M)
        b = np.stack([m.astype(np.float64) @ src[n].astype(np.float64) for n in range(N)])
        v0 += b @ Wt[:, k, :].T.astype(np.float64)
        term = dict(src=t(src), op=tp.add_operator(m), F=F, src_rows=M, src_stride=F, w=t(Wt[:, k, :].T), w_stride=ncols,
                    wT=Wt_d[:, k, :], wT_stride=K * F)
        if dual:
            v1 += b @ Wt2[:, k, :].T.astype(np.float64)
            term.update(w2=t(Wt2[:, k, :].T), w2_stride=ncols, w2T=Wt2_d[:, k, :], w2T_stride=K * F)
        terms.append(term)
    out = torch.full((N, M, ncols), float("nan"), device=dev)
    if dual:
        out2 = torch.full((N, M, ncols), float("nan"), device=dev)
        E.cheb_call(tp, N, M, ncols, terms, out, out2=out2, epilogue=E.EPI_AFFINE)
        torch.cuda.synchronize()
        assert _rel(out.cpu().numpy(), v1 + np.maximum(v0, 0)) < TOL
        assert _rel(out2.cpu().numpy(), np.maximum(v0, 0)) < TOL
    else:
        E.cheb_call(tp, N, M, ncols, terms, out)
        torch.cuda.synchronize()
        assert _rel(out.cpu().numpy(), v0) < TOL


# two accumulators, the second term without w2: its chunks add nothing to the second sum
@pytest.mark.parametrize("ncols", [64, 128])
def test_dual_term_without_second_weight(ncols):
    E, tp, dev = _ctx()
    rng = np.random.RandomState(5 + ncols)
    N, M = 16, 2200
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    v0 = np.zeros((N, M, ncols))
    v1 = np.zeros((N, M, ncols))
    terms = []
    for i, F in enumerate([96, 64]):
        src = rng.normal(size=(N, M, F)).astype(np.float32)
        m = _operator(rng, M)
        b = np.stack([m.astype(np.float64) @ src[n].astype(np.float64) for n in range(N)])
        w = rng.normal(0, 1 / np.sqrt(F), size=(F, ncols)).astype(np.float32)
        v0 += b @ w.astype(np.float64)
        term = dict(src=t(src), op=tp.add_operator(m), F=F, src_rows=M, src_stride=F, w=t(w), w_stride=ncols,
                    wT=t(w.T), wT_stride=F)
        if i == 0:
            w2 = rng.normal(0, 1 / np.sqrt(F), size=(F, ncols)).astype(np.float32)
            v1 += b @ w2.astype(np.float64)
            term.update(w2=t(w2), w2_stride=ncols, w2T=t(w2.T), w2T_stride=F)
        terms.append(term)
    out = torch.full((N, M, ncols), float("nan"), device=dev)
    out2 = torch.full((N, M, ncols), float("nan"), device=dev)
    E.cheb_call(tp, N, M, ncols, terms, out, out2=out2, epilogue=E.EPI_AFFINE)
    torch.cuda.synchronize()
    assert _rel(out.cpu().numpy(), v1 + np.maximum(v0, 0)) < TOL
    assert _rel(out2.cpu().numpy(), np.maximum(v0, 0)) < TOL


# BN = 128 from a captured graph three times and eagerly twice: the tensor maps captured by value, the tile counter at
# zero after every launch
def test_graph_replay_and_eager_launches_agree_wide():
    E, tp, dev = _ctx()
    rng = np.random.RandomState(8)
    N, M, F, ncols = 20, 2500, 96, 256
    m = _operator(rng, M)
    op = tp.add_operator(m)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    src = rng.normal(size=(N, M, F)).astype(np.float32)
    w = rng.normal(0, 1 / np.sqrt(F), size=(F, ncols)).astype(np.float32)
    terms = [dict(src=t(src), op=op, F=F, src_rows=M, src_stride=F, w=t(w), w_stride=ncols, wT=t(w.T), wT_stride=F)]
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
    assert _rel(first, want) < TOL
    for o in outs[1:]:
        assert np.array_equal(o.cpu().numpy(), first)
