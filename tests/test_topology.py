"""Host-side topology: fixtures, Laplacians vs the reference's own code (golden), operator algebra."""
import os

import numpy as np
import scipy.sparse as sp

from cape_b200 import topology as T

GOLD = os.path.join(os.path.dirname(__file__), "golden")


def test_fixture_invariants(hierarchy):
    """Facts of SURVEY.md section 0 / Appendix B that the kernels rely on."""
    h = hierarchy
    assert h["p"] == [6890, 6890, 3445, 3445, 1723, 1723, 862, 862, 862]
    assert [l.shape[0] for l in h["L_d"]] == [6890, 3445, 1723, 862, 431]
    for d in h["D"] + h["D_d"]:
        d = sp.csr_matrix(d)
        assert (np.diff(d.indptr) == 1).all() and (d.data == 1.0).all()      # pure row selection
        assert (np.diff(d.indices) > 0).all()                                # increasing columns
    for u in h["U"]:
        assert (np.diff(sp.csr_matrix(u).indptr) == 3).all()                 # 3-tap barycentric
    for i in (0, 2, 4, 6, 7):
        assert T.is_identity(h["D"][i], tol=0) and T.is_identity(h["U"][i], tol=1e-6)
    rs = np.asarray(h["U"][5].sum(1)).ravel()
    assert rs.min() < 0.95 and rs.max() > 1.02                               # row sums are NOT 1
    e = T.smpl_edges()
    assert e.shape == (20664, 2) and (e[:, 0] < e[:, 1]).all()


def test_laplacian_matches_reference_golden(hierarchy):
    from inputs import digest
    """laplacian + rescale_L reproduce the reference's lib/mesh_sampling.py output bit for bit."""
    z = np.load(os.path.join(GOLD, "lap_golden.npz"))
    for kind, Ls in (("for_demo", hierarchy["L"]), ("ds2", hierarchy["L_d"])):
        for i, L in enumerate(Ls):
            L = sp.csr_matrix(L)
            L.sort_indices()
            assert L.dtype == np.float32
            assert digest(L.indices) == str(z["%s.L.%d.indices" % (kind, i)])
            assert digest(L.data) == str(z["%s.L.%d.data" % (kind, i)])
            Lt = T.rescale_L(L, lmax=2)
            Lt.sort_indices()
            assert Lt.dtype == np.float32
            assert digest(Lt.indptr) == str(z["%s.Lt.%d.indptr" % (kind, i)])
            assert digest(Lt.indices) == str(z["%s.Lt.%d.indices" % (kind, i)])
            assert digest(Lt.data) == str(z["%s.Lt.%d.data" % (kind, i)])
            assert abs(Lt.diagonal()).max() == 0.0                           # zero diagonal (lmax = 2)


def test_rescale_does_not_modify_input(hierarchy):
    L = hierarchy["L"][0]
    before = L.copy()
    T.rescale_L(L)
    assert (L != before).nnz == 0


def _apply_ell(idx, w, x):
    y = np.zeros((idx.shape[0],) + x.shape[1:], np.float64)
    for j in range(idx.shape[1]):
        ok = idx[:, j] >= 0
        y[ok] += w[ok, j, None].astype(np.float64) * x[idx[ok, j]]
    return y


def test_composed_operator_equals_sequential(hierarchy):
    """D . T_k(L~) . U as one ELL gather == unpool -> Chebyshev recurrence -> pool."""
    h = hierarchy
    rng = np.random.RandomState(0)
    L, U, D = h["L"][2], h["U"][3], h["D"][3]           # unpool 1723 -> 3445, conv at 3445, pool -> 1723
    x = rng.normal(size=(U.shape[1], 5))
    Lt = T.rescale_L(L).astype(np.float64)
    z = U.astype(np.float64) @ x
    t0, t1 = z, Lt @ z
    t2 = 2 * (Lt @ t1) - t0
    Ts = T.cheb_polynomials(L, 3)
    for k, ref in enumerate((t0, t1, t2)):
        m = T.compose(D, Ts[k], U)
        idx, w = T.to_ell(m)
        got = _apply_ell(idx, w, x)
        want = D.astype(np.float64) @ ref
        assert np.abs(got - want).max() < 1e-5 * max(1.0, np.abs(want).max())
        # left-packed, -1 padded
        valid = idx >= 0
        assert (valid[:, :-1] >= valid[:, 1:]).all()


def test_adjacency_ell_counts_edges(hierarchy):
    idx, _ = T.adjacency_ell(hierarchy["L"][0])
    assert (idx >= 0).sum() == 2 * 20664


def _distinct_per_row(m, tile=128):
    m = sp.csr_matrix(m)
    r = [len(np.unique(m[r0:r0 + tile].indices)) / m[r0:r0 + tile].shape[0] for r0 in range(0, m.shape[0], tile)]
    return float(np.mean(r))


def test_patch_order_is_a_layout_change_only(hierarchy):
    """The internal vertex order: a permutation per level, coarse levels induced from the fine one, operators
    between re-ordered levels give the re-ordered result, and 128-row tiles touch fewer distinct rows."""
    h = hierarchy
    orders = T.level_orders(h["L"][0], h["D"])
    assert [len(o) for o in orders] == [l.shape[0] for l in h["L"]]
    for o in orders:
        assert np.array_equal(np.sort(o), np.arange(len(o)))
    assert T.patch_order(h["L"][0]) is orders[0]                 # cached, reproducible
    rng = np.random.RandomState(1)
    for lvl in (1, 3):                                           # a 2:1 pooled site and its unpool mirror
        m = T.compose(h["D"][lvl], T.cheb_polynomials(h["L"][lvl], 2)[1], None)
        oi, oo = orders[lvl], orders[lvl + 1]
        x = rng.normal(size=(m.shape[1], 3))
        assert np.abs(T.permute(m, oo, oi) @ x[oi] - (m @ x)[oo]).max() < 1e-12
        inv = T.inverse_order(oo)
        assert np.array_equal(oo[inv], np.arange(len(oo)))
        # induced order keeps the pooling a monotone selection
        sel = T.permute(h["D"][lvl], oo, oi).indices
        assert (np.diff(sel) > 0).all()
    Lt = T.rescale_L(h["L"][0])
    before, after = _distinct_per_row(Lt), _distinct_per_row(T.permute(Lt, orders[0], orders[0]))
    assert after < 0.75 * before and after < 1.7


def test_window_split_keeps_the_operator_and_packs_window_taps_first(hierarchy):
    h = hierarchy
    orders = T.level_orders(h["L"][0], h["D"])
    for lvl in (0, 6):
        Lt = T.cheb_polynomials(h["L"][lvl], 2)[1]
        for m in (Lt, T.permute(Lt, orders[lvl], orders[lvl])):
            idx, w, n_in = T.window_split(m, tile=128, halo=32)
            x = np.random.RandomState(0).normal(size=(m.shape[1], 2))
            assert np.abs(_apply_ell(idx, w, x) - m @ x).max() < 1e-5
            rows = np.arange(idx.shape[0])
            start = (rows // 128) * 128 - 32
            for j in range(idx.shape[1]):
                valid = idx[:, j] >= 0
                inwin = valid & (idx[:, j] - start >= 0) & (idx[:, j] - start < 192)
                assert np.array_equal(inwin, valid & (j < n_in))
        # patch order: almost every one-ring tap of a tile sits in its 192-row window
        idx, w, n_in = T.window_split(T.permute(Lt, orders[lvl], orders[lvl]))
        assert n_in.sum() / (idx >= 0).sum() > 0.85
