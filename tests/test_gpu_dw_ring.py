"""The wgmma weight-gradient kernel (dw_wg_kernel) on the shapes its producer/consumer ring has to get right, against a
float64 NumPy A^T . G: row splits whose chunks wrap the ring several times and end part-way through it, partial last
chunks, partial or half-used f tiles, partial last column tiles at 1-4 column tiles, accumulation into a strided dW
with and without split partials, a strided source with more source rows than output rows, and a gathered basis."""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

pytestmark = pytest.mark.gpu

TOL = 1e-4


def _operator(rng, rows_out, rows_in, width=7):
    """A random sparse [rows_out x rows_in] operator with `width` taps per row."""
    cols = rng.randint(0, rows_in, size=(rows_out, width))
    vals = rng.uniform(-1, 1, size=cols.shape)
    m = sp.csr_matrix((vals.ravel(), (np.repeat(np.arange(rows_out), width), cols.ravel())), shape=(rows_out, rows_in))
    m.sum_duplicates()
    return m.astype(np.float32)


def _rel(a, b):
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def run_case(N, M, ncols, F, gather=False, src_rows=None, src_stride=None, accumulate=False, K=1, k=0,
             workspace=True, seed=0):
    """dW (+)= sum_n (op . src[n][:, :F])^T . g[n], written to gW3[:, k, :] of a [F, K, ncols] buffer."""
    from cape_b200 import engine as E
    from cape_b200 import ops
    assert N * M >= 4096 and F % 4 == 0 and F >= 32 and ncols % 32 == 0 and 32 <= ncols <= 512, "not wgmma-eligible"
    dev = torch.device("cuda", 0)
    # a fresh handle has no workspace: every row goes into one split, reduced by the kernel's own epilogue
    tp = ops.topology_for(dev) if workspace else E.Topology(0)
    rng = np.random.RandomState(seed)
    src_rows = src_rows or M
    src_stride = src_stride or F
    src = rng.normal(size=(N, src_rows, src_stride)).astype(np.float32)
    g = rng.normal(size=(N, M, ncols)).astype(np.float32)
    if gather:
        m = _operator(rng, M, src_rows)
        op = tp.add_operator(m)
        basis = np.stack([m.astype(np.float64) @ src[n, :, :F].astype(np.float64) for n in range(N)])
    else:
        assert src_rows == M
        op, basis = -1, src[:, :, :F].astype(np.float64)
    want = np.einsum("nrf,nrc->fc", basis, g.astype(np.float64))
    gw3 = rng.normal(size=(F, K, ncols)).astype(np.float32)
    expect = gw3.astype(np.float64)
    if accumulate:
        expect[:, k, :] += want
    else:
        expect[:, k, :] = want
    gw3_d = torch.from_numpy(gw3).to(dev)
    E.cheb_dw(tp, N, M, ncols, torch.from_numpy(src).to(dev), op, F, src_rows, src_stride, torch.from_numpy(g).to(dev),
              gw3_d[:, k, :], K * ncols, accumulate=accumulate)
    torch.cuda.synchronize()
    got = gw3_d.cpu().numpy().astype(np.float64)
    assert _rel(got[:, k, :], expect[:, k, :]) < TOL
    others = [j for j in range(K) if j != k]
    assert np.array_equal(got[:, others, :], expect[:, others, :]), "wrote outside its dW slice"


# long row splits (5015 rows, a partial last chunk of 23 rows): the chunks of each split wrap the 5-, 4- or 3-stage
# ring several times; one split with no workspace, 160 chunks in one chain
@pytest.mark.parametrize("ncols", [32, 64, 128])
def test_ring_wraps(ncols):
    run_case(N=5, M=1003, ncols=ncols, F=160)
    run_case(N=5, M=1003, ncols=ncols, F=96, workspace=False)


# F of 32 and 64 (half of the f tile unused), 96 and 160 (partial f tile), 512 (four full f tiles)
@pytest.mark.parametrize("F", [32, 64, 96, 160, 512])
def test_f_tiles(F):
    run_case(N=3, M=1500, ncols=64, F=F)


# partial last column tile at 1 to 4 column tiles
@pytest.mark.parametrize("ncols", [32, 96, 160, 288, 480])
def test_column_tiles(ncols):
    run_case(N=2, M=2203, ncols=ncols, F=64)


# accumulate into gW3[:, k, :] (dw_stride = K * Fout): through reduce_splits, and through the kernel's epilogue
@pytest.mark.parametrize("workspace", [True, False])
def test_accumulate_strided(workspace):
    run_case(N=4, M=1111, ncols=96, F=128, accumulate=True, K=3, k=1, workspace=workspace)


# a strided source with more rows per sample than the output (the pooled layers' operators), gathered and plain
def test_strided_source():
    run_case(N=3, M=1400, ncols=160, F=64, gather=True, src_rows=2100, src_stride=72)
    run_case(N=3, M=1400, ncols=64, F=96, src_stride=100)


# gathered basis (the path with CAPE_DW_STASH=0)
@pytest.mark.parametrize("ncols", [64, 288])
def test_gathered_basis(ncols):
    run_case(N=3, M=1500, ncols=ncols, F=96, gather=True)
