"""The wgmma convolution kernel (conv_wg_kernel) on the shapes its producer/consumer ring has to get right, against a
float64 NumPy product: reductions that wrap the ring several times or end part-way through it, terms whose F changes
mid-ring, partial last row and column tiles, several samples per row tile with condition slots, the dual-accumulator
affine epilogue with a stash, and the slope / dual-mask data-gradient epilogues."""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

pytestmark = pytest.mark.gpu

TOL = 1e-4


def _operator(rng, rows, width=7):
    """A random sparse [rows x rows] operator with `width` taps per row (the diagonal among them)."""
    cols = np.concatenate([np.arange(rows)[:, None], rng.randint(0, rows, size=(rows, width - 1))], axis=1)
    vals = rng.uniform(-1, 1, size=cols.shape)
    m = sp.csr_matrix((vals.ravel(), (np.repeat(np.arange(rows), width), cols.ravel())), shape=(rows, rows))
    m.sum_duplicates()
    return m.astype(np.float32)


def _rel(a, b):
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def run_case(N, M, ncols, Fs, gather, dual=False, slots=0, epilogue="linear", stash=False, seed=0):
    from cape_b200 import engine as E
    from cape_b200 import ops
    dev = torch.device("cuda", 0)
    tp = ops.topology_for(dev)
    rng = np.random.RandomState(seed)
    C = 5
    cond = rng.normal(size=(N, C)).astype(np.float32) if slots else None
    terms, keep = [], []
    v0 = np.zeros((N, M, ncols))
    v1 = np.zeros((N, M, ncols))
    basis = []
    for i, (F, g) in enumerate(zip(Fs, gather)):
        src = rng.normal(size=(N, M, F)).astype(np.float32)
        if g:
            m = _operator(rng, M)
            op = tp.add_operator(m)
            b = np.stack([m.astype(np.float64) @ src[n].astype(np.float64) for n in range(N)])
            rowsum = np.asarray(m.astype(np.float64).sum(axis=1)).ravel()
        else:
            op, b, rowsum = -1, src.astype(np.float64), np.ones(M)
        basis.append(b)
        w = rng.normal(0, 1 / np.sqrt(F), size=(F, ncols)).astype(np.float32)
        t = dict(src=torch.from_numpy(src).to(dev), op=op, F=F, src_rows=M, src_stride=F,
                 w=torch.from_numpy(w).to(dev), w_stride=ncols, wT=torch.from_numpy(w.T.copy()).to(dev), wT_stride=F)
        v0 += b @ w.astype(np.float64)
        if dual:
            w2 = rng.normal(0, 1 / np.sqrt(F), size=(F, ncols)).astype(np.float32)
            t.update(w2=torch.from_numpy(w2).to(dev), w2_stride=ncols, w2T=torch.from_numpy(w2.T.copy()).to(dev),
                     w2T_stride=F)
            v1 += b @ w2.astype(np.float64)
        if i < slots:
            wc = rng.normal(size=(C, ncols)).astype(np.float32)
            t["wc"] = torch.from_numpy(wc).to(dev)
            v0 += rowsum[None, :, None] * (cond.astype(np.float64) @ wc.astype(np.float64))[:, None, :]
            if dual:
                wc2 = rng.normal(size=(C, ncols)).astype(np.float32)
                t["wc2"] = torch.from_numpy(wc2).to(dev)
                v1 += rowsum[None, :, None] * (cond.astype(np.float64) @ wc2.astype(np.float64))[:, None, :]
        if stash:
            t.update(stash=torch.full((N * M, F), float("nan"), device=dev), stash_stride=F)
        terms.append(t)
    out = torch.empty(N, M, ncols, device=dev)
    out2 = torch.empty(N, M, ncols, device=dev) if epilogue in ("affine", "dualmask") else None
    aux = rng.normal(size=(N, M, ncols)).astype(np.float32) if epilogue in ("slope", "dualmask") else None
    epi = {"linear": E.EPI_LINEAR, "affine": E.EPI_AFFINE, "slope": E.EPI_SLOPE, "dualmask": E.EPI_DUALMASK}[epilogue]
    E.cheb_call(tp, N, M, ncols, terms, out, out2=out2, epilogue=epi,
                cond=torch.from_numpy(cond).to(dev) if slots else None,
                aux=torch.from_numpy(aux).to(dev) if aux is not None else None, alpha=0.2)
    torch.cuda.synchronize()
    if epilogue == "linear":
        want = [v0]
    elif epilogue == "affine":
        want = [v1 + np.maximum(v0, 0), np.maximum(v0, 0)]
    elif epilogue == "slope":
        want = [v0 * np.where(aux > 0, 1.0, 0.2)]
    else:
        want = [v0, np.where(aux > 0, v0, 0.0)]
    got = [out] + ([out2] if out2 is not None else [])
    for g, w in zip(got, want):
        assert _rel(g.cpu().numpy(), w) < TOL
    if stash:
        for t, b in zip(terms, basis):
            assert _rel(t["stash"].cpu().numpy().reshape(N, M, -1), b) < TOL


# reductions of 14 and 10 chunks: several passes over a 3- or 4-stage ring, ending part-way through it
@pytest.mark.parametrize("ncols", [128, 64])
def test_ring_wraps(ncols):
    run_case(N=3, M=300, ncols=ncols, Fs=[224, 224], gather=[True, True])
    run_case(N=3, M=300, ncols=ncols, Fs=[160, 160], gather=[False, True])


# F changes between terms inside one pass over the ring, with partial last chunks (F % 32 != 0)
def test_terms_switch_mid_ring():
    run_case(N=2, M=257, ncols=128, Fs=[40, 72, 8, 100], gather=[True, False, True, True])


# partial last row tile (N * M % 128 != 0) and partial last column tile at 1 to 4 column tiles
@pytest.mark.parametrize("ncols", [96, 160, 288, 480])
def test_partial_tiles(ncols):
    run_case(N=2, M=203, ncols=ncols, Fs=[64, 64], gather=[True, True])


# up to four samples per 128-row tile, each with its condition vectors (qs)
@pytest.mark.parametrize("ncols", [32, 128])
def test_condition_slots(ncols):
    run_case(N=9, M=50, ncols=ncols, Fs=[64, 48], gather=[True, False], slots=2)


# the dual-accumulator affine epilogue, with condition slots on both accumulators and the basis stash
@pytest.mark.parametrize("ncols", [64, 128, 256])
def test_affine_dual_with_stash(ncols):
    run_case(N=3, M=90, ncols=ncols, Fs=[96, 96], gather=[False, True], dual=True, slots=1, epilogue="affine",
             stash=True)


@pytest.mark.parametrize("epilogue", ["slope", "dualmask"])
def test_data_gradient_epilogues(epilogue):
    run_case(N=2, M=211, ncols=160, Fs=[128, 128], gather=[True, True], epilogue=epilogue)
