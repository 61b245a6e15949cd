"""The wide tiles of the wgmma convolution kernel (conv_wg_kernel): a launch whose output spans more than one 128-row
tile's columns (ncols > 128) runs 64-row tiles of 256 columns (128 per sum with two accumulators), 16-deep
ring stages with the 64-byte swizzle and the two producer warpgroups filling alternate chunks.  Checked against a
float64 NumPy product by the harness of test_gpu_conv_ring.py, and for the tanh, TANHGRAD and pass-through cases by
one of the same kind here: partial row, column and k chunks, condition slots of tiles that straddle samples, the
stash, every epilogue, launches of many tiles per CTA, and graph replay against eager launches."""
import numpy as np
import pytest
import torch

from test_gpu_conv_ring import TOL, _operator, _rel, run_case

pytestmark = pytest.mark.gpu


# one to four wide column tiles, the last one partial at 160 and 288; F = 264 and 40 end part-way through a 16-deep
# stage and a 32-deep chunk, F = 20 part-way through the first stage
@pytest.mark.parametrize("ncols", [160, 256, 288, 512])
def test_widths(ncols):
    run_case(N=3, M=203, ncols=ncols, Fs=[264, 40, 20], gather=[True, False, True])


# the dual-accumulator affine epilogue (64 x 128 per sum) with condition slots on both sums and the basis stash,
# written by column tile 0 only
@pytest.mark.parametrize("ncols", [160, 256])
def test_affine_dual_with_stash(ncols):
    run_case(N=3, M=90, ncols=ncols, Fs=[96, 72], gather=[False, True], dual=True, slots=1, epilogue="affine",
             stash=True)


# rows_out = 50 and 203: a 64-row tile covers two or three samples, each with its condition vectors
@pytest.mark.parametrize("N,M,ncols", [(9, 50, 256), (300, 203, 288)])
def test_condition_slots(N, M, ncols):
    run_case(N=N, M=M, ncols=ncols, Fs=[64, 48], gather=[True, False], slots=2)


@pytest.mark.parametrize("epilogue", ["slope", "dualmask"])
def test_data_gradient_epilogues(epilogue):
    run_case(N=2, M=211, ncols=384, Fs=[128, 128], gather=[True, True], epilogue=epilogue)


# 825 row tiles x 2 column tiles over 132 SMs: the ring and the producers' chunk parity run on across tiles
def test_many_tiles():
    run_case(N=25, M=2111, ncols=512, Fs=[160, 96], gather=[True, False], stash=True)


def _conv(N, M, ncols, F, epilogue="linear", act="none", passthrough=False, seed=0):
    """One gathered term (+ an identity and a gathered pass-through term), checked against float64."""
    from cape_b200 import engine as E
    from cape_b200 import ops
    dev = torch.device("cuda", 0)
    tp = ops.topology_for(dev)
    rng = np.random.RandomState(seed)
    t = lambda a: torch.from_numpy(a).to(dev)
    src = rng.normal(size=(N, M, F)).astype(np.float32)
    m = _operator(rng, M)
    w = rng.normal(0, 1 / np.sqrt(F), size=(F, ncols)).astype(np.float32)
    terms = [dict(src=t(src), op=tp.add_operator(m), F=F, src_rows=M, src_stride=F, w=t(w), w_stride=ncols,
                  wT=t(w.T.copy()), wT_stride=F)]
    m64 = m.astype(np.float64)
    v = np.stack([m64 @ src[n].astype(np.float64) @ w.astype(np.float64) for n in range(N)])
    if passthrough:
        skip = rng.normal(size=(N, M, ncols)).astype(np.float32)
        ms = _operator(rng, M)
        skip2 = rng.normal(size=(N, M, ncols)).astype(np.float32)
        terms += [dict(src=t(skip), op=-1, F=ncols, src_rows=M, src_stride=ncols, w_stride=0),
                  dict(src=t(skip2), op=tp.add_operator(ms), F=ncols, src_rows=M, src_stride=ncols, w_stride=0)]
        v = v + skip + np.stack([ms.astype(np.float64) @ skip2[n] for n in range(N)])
    kw = {}
    if epilogue == "linear":
        bias = rng.normal(size=ncols).astype(np.float32)
        kw.update(bias=t(bias), act={"none": E.ACT_NONE, "tanh": E.ACT_TANH}[act])
        v = v + bias
        want = np.tanh(v) if act == "tanh" else v
    else:                                   # TANHGRAD: aux is the producing layer's tanh output y
        aux = np.tanh(rng.normal(size=(N, M, ncols))).astype(np.float32)
        kw.update(epilogue=E.EPI_TANHGRAD, aux=t(aux))
        want = v * (1 - aux.astype(np.float64) ** 2)
    out = torch.full((N, M, ncols), float("nan"), device=dev)
    E.cheb_call(tp, N, M, ncols, terms, out, **kw)
    torch.cuda.synchronize()
    assert _rel(out.cpu().numpy(), want) < TOL


@pytest.mark.parametrize("epilogue,act", [("linear", "tanh"), ("tanhgrad", "none")])
def test_tanh_epilogues(epilogue, act):
    _conv(N=3, M=203, ncols=288, F=136, epilogue=epilogue, act=act)


# pass-through terms (the encoder's residual skips at 256 and 512 columns), added in the epilogue
@pytest.mark.parametrize("ncols", [256, 512])
def test_pass_through(ncols):
    _conv(N=6, M=431, ncols=ncols, F=256, passthrough=True)


# one launch three times from a captured graph, and twice eagerly: every run draws its tiles from a counter at zero
def test_graph_replay_and_eager_launches_agree():
    from cape_b200 import engine as E
    from cape_b200 import ops
    dev = torch.device("cuda", 0)
    tp = ops.topology_for(dev)
    rng = np.random.RandomState(7)
    N, M, F, ncols = 20, 2500, 96, 256
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
    assert _rel(first, want) < TOL
    for o in outs[1:]:
        assert np.array_equal(o.cpu().numpy(), first)
