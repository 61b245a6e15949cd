"""The wgmma weight-gradient kernel (dw_wg_kernel) on the shapes its producer/consumer ring has to get right, against a
float64 A^T . G: row splits whose chunks wrap the ring several times and end part-way through it, partial last
chunks, partial or half-used f tiles, partial last column tiles at 1-4 column tiles, accumulation into a strided dW
with and without split partials, a strided source with more source rows than output rows, and a gathered basis.

Long accumulation chains (test_long_chains, test_single_chain_65k).  The tensor core's fp32 accumulation truncates,
so a sum over one long chain of MMAs shrinks a little with every MMA; in a split of more than 64 chunks the kernel
ends a chain every 64 chunks (2048 rows) by adding its accumulators into its output slice in fp32.  The split plan
aims at two waves of CTAs, so the rows
per split grow with the batch: about 1.7k rows at batch 64, 6.7k at 256, 13.4k at 512 and 26.8k at 1024 for the
network's layer shapes (test_split_plan_rows).  The cases force those chain lengths on one set of operands per shape by
giving a fresh handle workspace for exactly k partials, for every column tile width (32, 64, 128, 256; one case with
four f tiles and two column tiles), plain and gathered bases, and three operand regimes:
  - "zero-mean": A and G N(0, 1); the products have zero mean, so truncation errors cancel like a random walk;
  - "relu": A = leaky_relu(N(0.5, 1)), like an activation, against a zero-mean G;
  - "coherent": the same A against G = N(0.25, 1); the products have a mean, and so has the truncation error.
Each case prints, per chain length, max|e| / max|truth| and the signed bias mean(e sign(truth)) / mean|truth| of the
kernel, of the same kernel with one MMA chain per split (cape_set_tuning(11, -1), what it did before chains were
bounded), and max|e| / max|truth| of the fp32 kernel (tensor cores off) on the same inputs.  Asserted: the kernel and
the fp32 kernel within 1e-4 everywhere, and the kernel's error at the longest chain at most twice its error at the
batch-64 chain.  Measured on an H100 SXM (700 W): the single chain loses 1.1e-5 .. 1.6e-5 at 1.7k rows, 1.6e-4 ..
2.7e-4 at 27.6k and 5e-4 at 68.9k, with a signed bias of about minus its error in every regime; the bounded chains
1.1e-5 .. 2.0e-5 at every length (DESIGN.md section 2)."""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

gpu = pytest.mark.gpu

TOL = 1e-4
REGIMES = ("zero-mean", "relu", "coherent")


def _operator(rng, rows_out, rows_in, width=7, positive=False):
    """A random sparse [rows_out x rows_in] operator with `width` taps per row (weights in [0, 1) if positive, like a
    pooling operator's: the gathered basis then keeps the mean of the source)."""
    cols = rng.randint(0, rows_in, size=(rows_out, width))
    vals = rng.uniform(0 if positive else -1, 1, size=cols.shape)
    m = sp.csr_matrix((vals.ravel(), (np.repeat(np.arange(rows_out), width), cols.ravel())), shape=(rows_out, rows_in))
    m.sum_duplicates()
    return m.astype(np.float32)


def _operands(rng, N, M, src_rows, src_stride, ncols, regime):
    """src [N, src_rows, src_stride] and g [N, M, ncols] (float32) of one operand regime."""
    if regime == "zero-mean":
        return (rng.normal(size=(N, src_rows, src_stride)).astype(np.float32),
                rng.normal(size=(N, M, ncols)).astype(np.float32))
    a = rng.normal(0.5, 1.0, size=(N, src_rows, src_stride))
    a = np.where(a > 0, a, 0.2 * a).astype(np.float32)
    return a, rng.normal(0.25 if regime == "coherent" else 0.0, 1.0, size=(N, M, ncols)).astype(np.float32)


def _truth(src, g, F, m=None):
    """float64 sum_n B[n]^T . g[n] with B[n] = (m .) src[n][:, :F], as one BLAS product over all rows."""
    N, ncols = g.shape[0], g.shape[2]
    if m is None:
        basis = src[:, :, :F].astype(np.float64)
    else:
        m64 = m.astype(np.float64)
        basis = np.stack([m64 @ src[n, :, :F].astype(np.float64) for n in range(N)])
    return basis.reshape(-1, F).T @ g.reshape(-1, ncols).astype(np.float64)


def _split_rows(total_rows, F, ncols, workspace_bytes, sms):
    """Rows per split (the MMA chain before chains were bounded) of launch_ellconv_dw_tc's split plan."""
    bn = 32 if ncols <= 32 else 64 if ncols <= 64 else 128 if ncols <= 128 else 256
    tiles = -(-F // 128) * -(-ncols // bn)
    nsplit = min(-(-2 * sms // tiles), -(-total_rows // 512))
    per = F * ncols * 4
    if nsplit > 1 and nsplit * per > workspace_bytes:
        nsplit = workspace_bytes // per
    nsplit = max(nsplit, 1)
    rps = -(-total_rows // nsplit)
    return -(-rps // 32) * 32


def _errors(got, want):
    """max|e| / max|truth| and the signed bias mean(e sign(truth)) / mean|truth|."""
    e = got - want
    return float(np.abs(e).max() / max(np.abs(want).max(), 1e-30)), float(
        (e * np.sign(want)).mean() / max(np.abs(want).mean(), 1e-30))


def _rel(a, b):
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def run_case(N, M, ncols, F, gather=False, src_rows=None, src_stride=None, accumulate=False, K=1, k=0,
             workspace=True, seed=0, regime="zero-mean", splits=None):
    """dW (+)= sum_n (op . src[n][:, :F])^T . g[n], written to gW3[:, k, :] of a [F, K, ncols] buffer.

    regime: the operands (REGIMES).  splits: None runs the case once, on the network's handle (64 MB of workspace) or,
    workspace=False, on a fresh one without workspace (one split, reduced by the kernel's own epilogue).  A list of
    split counts runs it once per count on a fresh handle with workspace for exactly that many partials, and also on
    the fp32 kernel and with one MMA chain per split; it returns one row per count: the split's rows and the errors."""
    from cape_b200 import engine as E
    from cape_b200 import ops
    import test_gpu_thin_paths as TP
    assert N * M >= 4096 and F % 4 == 0 and F >= 32 and ncols % 32 == 0 and 32 <= ncols <= 512, "not wgmma-eligible"
    dev = torch.device("cuda", 0)
    rng = np.random.RandomState(seed)
    src_rows = src_rows or M
    src_stride = src_stride or F
    src, g = _operands(rng, N, M, src_rows, src_stride, ncols, regime)
    assert gather or src_rows == M
    m = _operator(rng, M, src_rows, positive=regime != "zero-mean") if gather else None
    want = _truth(src, g, F, m)
    gw3 = rng.normal(size=(F, K, ncols)).astype(np.float32)
    expect = gw3.astype(np.float64)
    if accumulate:
        expect[:, k, :] += want
    else:
        expect[:, k, :] = want
    src_d, g_d = torch.from_numpy(src).to(dev), torch.from_numpy(g).to(dev)

    def launch(tp, tc=True, tuning=()):
        op = tp.add_operator(m) if gather else -1
        gw3_d = torch.from_numpy(gw3).to(dev)
        with TP._knobs(tuning=tuning, tc=tc):
            E.cheb_dw(tp, N, M, ncols, src_d, op, F, src_rows, src_stride, g_d, gw3_d[:, k, :], K * ncols,
                      accumulate=accumulate)
        torch.cuda.synchronize()
        got = gw3_d.cpu().numpy().astype(np.float64)
        others = [j for j in range(K) if j != k]
        assert np.array_equal(got[:, others, :], expect[:, others, :]), "wrote outside its dW slice"
        return got[:, k, :]

    if splits is None:
        # a fresh handle has no workspace: every row goes into one split, reduced by the kernel's own epilogue
        assert _rel(launch(ops.topology_for(dev) if workspace else E.Topology(0)), expect[:, k, :]) < TOL
        return None
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    rows = []
    for s in splits:
        ws = s * F * ncols * 4 if s > 1 else 0

        def fresh():
            tp = E.Topology(0)
            if ws:
                tp.reserve_workspace(ws)
            return tp
        r = dict(splits=s, rows=_split_rows(N * M, F, ncols, ws, sms),
                 tc=_errors(launch(fresh()), expect[:, k, :]),
                 one_chain=_errors(launch(fresh(), tuning=((11, -1),)), expect[:, k, :]),
                 fp32=_errors(launch(fresh(), tc=False), expect[:, k, :]))
        rows.append(r)
    return rows


def _table(label, rows):
    print("\n%s\n  %6s %7s  %10s %10s  %14s %14s  %10s" % (label, "splits", "chain", "tc err", "tc bias",
                                                          "1-chain err", "1-chain bias", "fp32 err"))
    for r in rows:
        print("  %6d %7d  %10.2e %+10.2e  %14.2e %+14.2e  %10.2e" % (
            r["splits"], r["rows"], r["tc"][0], r["tc"][1], r["one_chain"][0], r["one_chain"][1], r["fp32"][0]))


def _assert_chains(label, rows):
    """Every chain within TOL (tensor cores and fp32); the longest chain's error at most twice the shortest's."""
    bad = [r for r in rows if not (r["tc"][0] < TOL and r["fp32"][0] < TOL)]
    assert not bad, "%s: %s" % (label, bad)
    assert rows[-1]["tc"][0] <= 2 * rows[0]["tc"][0], "%s: error grows with the chain: %s" % (label, rows)


# long row splits (5015 rows, a partial last chunk of 23 rows): the chunks of each split wrap the 5-, 4- or 3-stage
# ring several times; one split with no workspace, 160 chunks in one chain
@gpu
@pytest.mark.parametrize("ncols", [32, 64, 128])
def test_ring_wraps(ncols):
    run_case(N=5, M=1003, ncols=ncols, F=160)
    run_case(N=5, M=1003, ncols=ncols, F=96, workspace=False)


# F of 32 and 64 (half of the f tile unused), 96 and 160 (partial f tile), 512 (four full f tiles)
@gpu
@pytest.mark.parametrize("F", [32, 64, 96, 160, 512])
def test_f_tiles(F):
    run_case(N=3, M=1500, ncols=64, F=F)


# partial last column tile at 1 to 4 column tiles
@gpu
@pytest.mark.parametrize("ncols", [32, 96, 160, 288, 480])
def test_column_tiles(ncols):
    run_case(N=2, M=2203, ncols=ncols, F=64)


# accumulate into gW3[:, k, :] (dw_stride = K * Fout): through reduce_splits, and through the kernel's epilogue
@gpu
@pytest.mark.parametrize("workspace", [True, False])
def test_accumulate_strided(workspace):
    run_case(N=4, M=1111, ncols=96, F=128, accumulate=True, K=3, k=1, workspace=workspace)


# a strided source with more rows per sample than the output (the pooled layers' operators), gathered and plain
@gpu
def test_strided_source():
    run_case(N=3, M=1400, ncols=160, F=64, gather=True, src_rows=2100, src_stride=72)
    run_case(N=3, M=1400, ncols=64, F=96, src_stride=100)


# gathered basis (the path with CAPE_DW_STASH=0)
@gpu
@pytest.mark.parametrize("ncols", [64, 288])
def test_gathered_basis(ncols):
    run_case(N=3, M=1500, ncols=ncols, F=96, gather=True)


# several bounded chains in one split, added into dW (accumulating: every chain adds) or stored then added: 4 x 1100
# rows = 137 full chunks + 16 rows, so chains of 64 chunks and a last one of 10 that ends in a partial chunk
@gpu
@pytest.mark.parametrize("ncols", [64, 288])
def test_bounded_chains_one_split(ncols):
    run_case(N=4, M=1100, ncols=ncols, F=96, gather=True, accumulate=True, K=3, k=2, workspace=False,
             regime="coherent")
    run_case(N=4, M=1100, ncols=ncols, F=96, workspace=False, regime="coherent")


# the network's layer shapes (output rows, F = ncols as in the split-plan table; ncols 32 at the 6890-row level, and
# F 512 with 512 columns: four f tiles, two column tiles of 256) at about 27.6k rows, so that 16, 4, 2 and 1 splits
# give the chains of batch 64, 256, 512 and 1024
LONG = [(32, 64, 6890, 4), (64, 64, 6890, 4), (128, 128, 3445, 8), (256, 256, 1723, 16), (512, 512, 862, 32)]


@gpu
@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("gather", [False, True], ids=["plain", "gathered"])
@pytest.mark.parametrize("ncols,F,M,N", LONG, ids=["c%d" % c for c, *_ in LONG])
def test_long_chains(ncols, F, M, N, gather, regime):
    label = "dW chains: %d rows x F %d x %d columns, %s basis, %s operands" % (N * M, F, ncols,
                                                                               "gathered" if gather else "plain", regime)
    rows = run_case(N=N, M=M, ncols=ncols, F=F, gather=gather, regime=regime, splits=(16, 4, 2, 1), seed=1)
    _table(label, rows)
    _assert_chains(label, rows)


# one split of 68,900 rows (10 x the 6890-row level), against 40 splits of 1728 rows (batch 64's chain)
@gpu
@pytest.mark.parametrize("regime", REGIMES)
def test_single_chain_65k(regime):
    label = "dW chains: 68900 rows x F 64 x 64 columns, plain basis, %s operands" % regime
    rows = run_case(N=10, M=6890, ncols=64, F=64, regime=regime, splits=(40, 1), seed=2)
    _table(label, rows)
    assert rows[-1]["rows"] >= 65536
    _assert_chains(label, rows)


# ---- CPU: the truth, the operands and the split plan the long-chain cases rely on --------------------------------------
def test_split_plan_rows():
    """The rows per split (one MMA chain before chains were bounded) of the network's layer shapes, H100 (132 SMs) and
    the network's 64 MB workspace, at batch 64 .. 1024."""
    want = {(6890, 64): [1696, 6688, 13376, 26752], (3445, 128): [864, 3360, 6688, 13376],
            (1723, 256): [864, 3360, 6688, 13376], (862, 512): [1696, 6688, 13376, 26752]}
    for (rows, f), chains in want.items():
        assert [_split_rows(n * rows, f, f, 64 << 20, 132) for n in (64, 256, 512, 1024)] == chains, (rows, f)
    # the forced split counts of the long-chain cases
    assert [_split_rows(27560, 64, 64, k * 64 * 64 * 4 if k > 1 else 0, 132) for k in (16, 4, 2, 1)] == \
        [1728, 6912, 13792, 27584]
    assert _split_rows(68900, 64, 64, 0, 132) == 68928


@pytest.mark.parametrize("gather", [False, True])
def test_truth_and_regimes(gather):
    """_truth against a per-row einsum in float64, plain and gathered, and the means of the three regimes."""
    rng = np.random.RandomState(3)
    N, M, src_rows, F, ncols = 3, 40, 50 if gather else 40, 12, 8
    for regime in REGIMES:
        src, g = _operands(rng, N, M, src_rows, F + 4, ncols, regime)
        assert src.dtype == np.float32 and g.dtype == np.float32
        m = _operator(rng, M, src_rows, positive=regime != "zero-mean") if gather else None
        basis = src[:, :, :F].astype(np.float64)
        if gather:
            basis = np.einsum("rs,nsf->nrf", m.toarray().astype(np.float64), basis)
        want = np.einsum("nrf,nrc->fc", basis, g.astype(np.float64))
        assert np.allclose(_truth(src, g, F, m), want, rtol=1e-12, atol=1e-12)
    big_a, big_g = _operands(np.random.RandomState(4), 4, 4096, 4096, 32, 32, "coherent")
    assert 0.62 < big_a.mean() < 0.7 and 0.2 < big_g.mean() < 0.3     # E leaky_relu(N(0.5, 1)) = 0.658
    assert abs(_operands(np.random.RandomState(4), 4, 4096, 4096, 32, 32, "relu")[1].mean()) < 0.01
