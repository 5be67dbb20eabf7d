"""kron_reduction(method='walks') on the device (pygsp_b200/reduction.py _schur_walks,
csrc/schur_walk.cu): the samples against the NumPy restatement with the same draws
(oracle/schur_walks_oracle.py), determinism and symmetry, the statistics against the exact path,
the errors, and graph_multiresolution with walks and sketched resistances at 10^4 and 10^5
vertices."""
import time

import numpy as np
import pytest
from scipy import sparse

from oracle import schur_walks_oracle as swo

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gsp():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import pygsp_b200
    return pygsp_b200


def _split(G):
    V = G._largest_eigenvector(seed=0)
    V *= np.sign(V[0])
    return np.nonzero(V >= 0)[0]


def _host_l(G):
    return G.L.to_scipy().astype(np.float64).tocsr()


def _two_components_and_a_dead_one():
    """Two grids joined by nothing, and a path whose vertices are all removed."""
    def grid(k, w0):
        n = k * k
        rows, cols = [], []
        for i in range(k):
            for j in range(k):
                v = i * k + j
                if j + 1 < k:
                    rows.append(v), cols.append(v + 1)
                if i + 1 < k:
                    rows.append(v), cols.append(v + k)
        w = w0 * (1.0 + np.arange(len(rows)) % 3)
        W = sparse.coo_matrix((w, (rows, cols)), shape=(n, n))
        return (W + W.T).tocsr()
    path = sparse.diags([np.ones(5), np.ones(5)], [-1, 1], shape=(6, 6))
    W = sparse.block_diag([grid(5, 1.0), grid(4, 0.5), path]).tocsr()
    L = (sparse.diags(np.asarray(W.sum(axis=1)).ravel()) - W).tocsr()
    ind = np.r_[np.arange(0, 25, 3), np.arange(25, 41, 5)]
    return L, ind


def _device_walks(gsp, M, ind, samples, key, excess=None):
    import torch
    red = gsp.reduction
    _, dev = red._ctx()
    Md = red._device_matrix(M, dev)
    ex = None if excess is None else torch.full((M.shape[0],), float(excess), dtype=torch.float64,
                                                device=dev)
    return red._schur_walks(Md, np.asarray(ind, dtype=np.int64), samples, key, 2 ** 20,
                            excess=ex).to_scipy()


def _assert_same(got, want):
    got, want = sparse.csr_matrix(got), sparse.csr_matrix(want)
    got.sort_indices()
    want.sort_indices()
    np.testing.assert_array_equal(got.indptr, want.indptr)
    np.testing.assert_array_equal(got.indices, want.indices)
    rel = np.abs(got.data - want.data) / np.abs(want.data)
    print("structure equal, %d entries, max relative difference %.2e" % (want.nnz, rel.max()))
    assert rel.max() <= 1e-14


def _case(gsp, name):
    """(M, ind, excess) -- excess None: derived from M (the matrix branch)."""
    if name == "grid12":
        G = gsp.graphs.Grid2d(12, dtype=np.float64)
        return _host_l(G), _split(G), 0.0
    if name in ("sensor500", "sensor500_f32"):
        G = gsp.graphs.Sensor(500, k=10, seed=2,
                              dtype=np.float32 if name.endswith("f32") else np.float64)
        return _host_l(G), _split(G), 0.0
    if name == "matrix_reg":
        G = gsp.graphs.Sensor(500, k=10, seed=2, dtype=np.float64)
        return (_host_l(G) + 0.005 * sparse.eye(G.N)).tocsr(), _split(G), None
    return (*_two_components_and_a_dead_one(), None)


@pytest.mark.parametrize("samples", [1, 3])
@pytest.mark.parametrize("name", ["grid12", "sensor500", "sensor500_f32", "matrix_reg",
                                  "dead_component"])
def test_device_equals_oracle(gsp, name, samples):
    M, ind, excess = _case(gsp, name)
    key = gsp.reduction._sampling_seed(4, 1 << 21)
    got = _device_walks(gsp, M, ind, samples, key, excess)
    want = swo.schur_walks(M, ind, samples, key, excess=excess)
    _assert_same(got, want)


def test_public_branches_equal_oracle(gsp):
    """kron_reduction(G, method='walks') is -offdiag of the sampled reduction with excess 0; the
    matrix branch returns the sampled L_new with its diagonal."""
    G = gsp.graphs.Sensor(500, k=10, seed=2, dtype=np.float64)
    ind = _split(G)
    L = _host_l(G)
    key = gsp.reduction._sampling_seed(9, 1 << 21)
    H = swo.schur_walks(L, ind, 16, key, excess=0.0)
    Gr = gsp.reduction.kron_reduction(G, ind, method="walks", seed=9)
    assert Gr.N == len(ind) and Gr.dtype == G.dtype
    np.testing.assert_array_equal(Gr.coords, G.coords[ind])
    W = -(H - sparse.diags(H.diagonal()))
    W.eliminate_zeros()
    _assert_same(Gr.W.to_scipy(), W)
    Lreg = (L + 0.005 * sparse.eye(G.N)).tocsr()
    got = gsp.reduction.kron_reduction(Lreg, ind, method="walks", seed=9)
    assert sparse.isspmatrix_csr(got) and got.dtype == np.float64
    _assert_same(got, swo.schur_walks(Lreg, ind, 16, key))


def test_determinism_and_symmetry(gsp):
    import torch
    G = gsp.graphs.Sensor(2000, k=10, seed=3, order="morton")
    ind = _split(G)
    A = gsp.reduction.kron_reduction(G, ind, method="walks", seed=5)
    B = gsp.reduction.kron_reduction(G, ind, method="walks", seed=5)
    C = gsp.reduction.kron_reduction(G, ind, method="walks", seed=6)
    for a, b in ((A.W.indptr, B.W.indptr), (A.W.indices, B.W.indices), (A.W.data, B.W.data)):
        assert torch.equal(a, b)
    assert not (A.W.indptr.shape == C.W.indptr.shape and torch.equal(A.W.indptr, C.W.indptr)
                and torch.equal(A.W.indices, C.W.indices) and torch.equal(A.W.data, C.W.data))
    assert not A.is_directed()
    L = _host_l(gsp.graphs.Sensor(2000, k=10, seed=3, order="morton", dtype=np.float64))
    H = gsp.reduction.kron_reduction((L + 0.005 * sparse.eye(L.shape[0])).tocsr(), ind,
                                     method="walks", seed=5)
    assert abs(H - H.T).max() == 0


def test_mean_over_seeds_is_the_exact_reduction(gsp):
    """The mean over 200 seeds against the exact path, within 5 standard errors from the sample
    variance: every entry whose sampled part is nonzero for at least 20 seeds, and 32 random
    quadratic forms.  The exact reduction is dense in each component, and most of its small
    entries are hit by a few seeds or none, where a sample variance says nothing."""
    G = gsp.graphs.Sensor(200, k=10, seed=4, dtype=np.float64)
    L = _host_l(G)
    ind = _split(G)
    SC = gsp.reduction.kron_reduction(L, ind).toarray()
    Y = np.stack([gsp.reduction.kron_reduction(L, ind, method="walks", seed=s).toarray()
                  for s in range(200)])
    K = L[ind][:, ind].toarray()
    np.fill_diagonal(K, 0)                           # the exact samples off the diagonal
    well = ((Y - K) != 0).sum(axis=0) >= 20
    mean, se = Y.mean(axis=0), Y.std(axis=0, ddof=1) / np.sqrt(len(Y))
    scale = np.abs(SC).max()
    z = np.abs(mean - SC) / np.maximum(se, 1e-300)
    print("largest |mean - exact| / se over %d well-sampled entries: %.2f" % (well.sum(),
                                                                              z[well].max()))
    assert well.sum() >= 1000
    assert np.all((np.abs(mean - SC) <= 5 * se + 1e-10 * scale)[well])
    X = np.random.default_rng(0).standard_normal((len(ind), 32))
    q = np.einsum("ij,sik,kj->sj", X, Y, X)
    qx = np.einsum("ij,ik,kj->j", X, SC, X)
    zq = np.abs(q.mean(axis=0) - qx) / (q.std(axis=0, ddof=1) / np.sqrt(len(Y)))
    print("largest quadratic-form |mean - exact| / se: %.2f" % zq.max())
    assert zq.max() <= 5


def test_spectrum_against_the_exact_path(gsp):
    G = gsp.graphs.Sensor(3000, k=10, seed=1, dtype=np.float64, order="morton")
    L = _host_l(G)
    ind = _split(G)
    SC = gsp.reduction.kron_reduction(L, ind).toarray()
    H = gsp.reduction.kron_reduction(L, ind, method="walks", seed=1)
    lo, hi = swo.generalized_spread(H.toarray(), SC)
    print("Sensor(3000): %d kept, spread [%.3f, %.3f], entries %d (exact %d)"
          % (len(ind), lo, hi, H.nnz, np.count_nonzero(SC)))
    assert 0.8 <= lo and hi <= 1.25


def test_errors(gsp):
    red = gsp.reduction
    G = gsp.graphs.Sensor(200, k=6, seed=3, dtype=np.float64)
    ind = np.arange(0, 200, 2)
    with pytest.raises(ValueError, match="method"):
        red.kron_reduction(G, ind, method="dense")
    with pytest.raises(ValueError, match="samples"):
        red.kron_reduction(G, ind, method="walks", samples=0)
    with pytest.raises(ValueError, match="method"):
        red.graph_multiresolution(G, 1, kron_method="dense")
    L = _host_l(G).tolil()
    L[0, 1] -= 0.25                                    # asymmetric
    with pytest.raises(ValueError, match="symmetric"):
        red.kron_reduction(L.tocsr(), ind, method="walks")
    L = _host_l(G).tolil()
    j = next(c for c in L.rows[0] if c != 0)
    L[0, j] = L[j, 0] = 0.5                            # a negative weight
    with pytest.raises(ValueError, match="non-negative"):
        red.kron_reduction(L.tocsr(), ind, method="walks")
    L = _host_l(G).tolil()
    L[1, 1] = 0.5 * L[1, 1]                            # not diagonally dominant
    with pytest.raises(ValueError, match="diagonally dominant"):
        red.kron_reduction(L.tocsr(), ind, method="walks")
    P = gsp.graphs.Path(50, dtype=np.float64)
    with pytest.raises(ValueError, match="max_steps"):
        red.kron_reduction(P, [0, 49], method="walks", max_steps=10)
    # the same call with room to walk completes: a single edge of the series conductance
    Pr = red.kron_reduction(P, [0, 49], method="walks", samples=64)
    assert Pr.N == 2 and Pr.W.nnz == 2


def _check_levels(Gs):
    for i, g in enumerate(Gs):
        assert g.is_connected()
        assert not g.is_directed()
        if i:
            assert g.N < Gs[i - 1].N and g.mr["level"] == i - 1
            assert sparse.isspmatrix_csr(Gs[i - 1].mr["K_reg"])
            assert Gs[i - 1].mr["K_reg"].shape == (g.N, g.N)


def test_pipeline_at_1e4(gsp):
    import torch
    kw = dict(kron_method="walks", resistances="sketch")
    G = gsp.graphs.Sensor(10_000, k=10, seed=1, order="morton")
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    Gs = gsp.reduction.graph_multiresolution(G, 3, **kw)
    torch.cuda.synchronize()
    print("graph_multiresolution(Sensor(1e4), 3, walks, sketch): %.2f s, N = %s, nnz = %s"
          % (time.perf_counter() - t0, [g.N for g in Gs], [g.W.nnz for g in Gs]))
    assert len(Gs) == 4
    _check_levels(Gs)
    again = gsp.reduction.graph_multiresolution(
        gsp.graphs.Sensor(10_000, k=10, seed=1, order="morton"), 3, **kw)
    for g, h in zip(Gs, again):
        for a, b in ((g.W.indptr, h.W.indptr), (g.W.indices, h.W.indices), (g.W.data, h.W.data)):
            assert torch.equal(a, b)
        np.testing.assert_array_equal(g.mr["idx"], h.mr["idx"])
    for g, h in zip(Gs[:-1], again[:-1]):
        assert (g.mr["K_reg"] != h.mr["K_reg"]).nnz == 0
    f = np.random.default_rng(0).standard_normal((G.N, 1))
    ca, pe = gsp.reduction.pyramid_analysis(Gs, f, order=30)
    rec, _ = gsp.reduction.pyramid_synthesis(Gs, ca[3], pe, order=30)
    assert np.linalg.norm(rec - f) / np.linalg.norm(f) <= 1e-5


def test_pipeline_at_1e5(gsp):
    import torch
    free, _ = torch.cuda.mem_get_info()
    if free < 16 * 2 ** 30:
        pytest.skip("needs 16 GB of free device memory")
    G = gsp.graphs.Sensor(100_000, k=10, seed=1, order="morton")
    with pytest.raises(ValueError):
        gsp.reduction.graph_multiresolution(G, 3)
    G = gsp.graphs.Sensor(100_000, k=10, seed=1, order="morton")
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    Gs = gsp.reduction.graph_multiresolution(G, 3, kron_method="walks", resistances="sketch")
    torch.cuda.synchronize()
    print("graph_multiresolution(Sensor(1e5), 3, walks, sketch): %.2f s, N = %s, nnz = %s"
          % (time.perf_counter() - t0, [g.N for g in Gs], [g.W.nnz for g in Gs]))
    assert len(Gs) == 4
    _check_levels(Gs)
