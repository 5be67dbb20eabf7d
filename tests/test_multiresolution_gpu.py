"""graph_multiresolution, kron_reduction, graph_sparsify and resistance_distance on the device
(pygsp_b200/reduction.py, csrc/schur.cu) against the fixtures of the unmodified PyGSP 0.6.1
(tests/golden/pyramid.npz, tests/golden/multiresolution.npz) and dense float64 restatements."""
import numpy as np
import pytest
from scipy import sparse, stats

from conftest import csr_from
from oracle import multiresolution_oracle as mro
from oracle.pygsp_oracle import laplacian

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gsp():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import pygsp_b200
    return pygsp_b200


def _rowwise(got, want):
    """max over rows of max|got - want| / max|want| (the row's largest weight)."""
    got, want = np.asarray(got), np.asarray(want)
    scale = np.maximum(np.abs(want).max(axis=1), 1e-300)
    return float((np.abs(got - want).max(axis=1) / scale).max())


def _same_pattern(got, want):
    """Patterns equal, or differing only by entries below 1e-12 of their row's maximum."""
    got, want = np.asarray(got), np.asarray(want)
    scale = np.maximum(np.abs(want).max(axis=1, keepdims=True), 1e-300)
    differ = (got != 0) != (want != 0)
    small = np.maximum(np.abs(got), np.abs(want)) <= 1e-12 * scale
    return bool(np.all(~differ | small))


DTYPES = [(np.float64, 1e-10), (np.float32, 2e-6)]


@pytest.mark.parametrize("dtype,tol", DTYPES)
def test_multiresolution_matches_pyramid_fixture(gsp, golden, dtype, tol):
    z = golden("pyramid")
    levels = int(z["levels"])
    G = gsp.graphs.Graph(csr_from(z, "W0"), dtype=dtype)
    Gs = gsp.reduction.graph_multiresolution(G, levels, sparsify=False)
    assert len(Gs) == levels + 1
    for i in range(1, levels + 1):
        np.testing.assert_array_equal(Gs[i].mr["idx"], z["idx%d" % i])
        assert Gs[i].mr["level"] == i - 1
        np.testing.assert_array_equal(Gs[i].mr["orig_idx"],
                                      Gs[i - 1].mr["orig_idx"][z["idx%d" % i]])
        got, want = Gs[i].W.toarray(), csr_from(z, "W%d" % i).toarray()
        assert _rowwise(got, want) <= tol
        assert _same_pattern(got, want)
        assert not Gs[i].is_directed()
    for i in range(levels):
        np.testing.assert_allclose(Gs[i].mr["K_reg"].toarray(), z["Kreg%d" % i], rtol=1e-6,
                                   atol=1e-8)

    # the pyramid on the engine-built graphs, with the fixture's lmax
    for i, g in enumerate(Gs):
        g._lmax, g._lmax_method = float(z["lmax%d" % i]), "lanczos"
    order = int(z["order"])
    h = [lambda x: 5.0 / (5 + x)]
    ptol = 1e-7 if dtype == np.float64 else 5e-4
    ca, pe = gsp.reduction.pyramid_analysis(Gs, z["f"], h_filters=h, order=order)
    scale = np.abs(z["f"]).max()
    for i in range(levels + 1):
        assert np.abs(ca[i] - z["ca%d" % i]).max() <= ptol * scale
    for i in range(levels):
        assert np.abs(pe[i] - z["pe%d" % i]).max() <= ptol * scale
    rec, _ = gsp.reduction.pyramid_synthesis(Gs, ca[levels], pe, order=order)
    assert np.abs(rec - z["reconstruction"]).max() <= ptol * scale


def test_multiresolution_matches_grid_fixture(gsp, golden):
    z = golden("multiresolution")
    levels = int(z["mr_levels"])
    G = gsp.graphs.Graph(csr_from(z, "mr_W0"), dtype=np.float64)
    Gs = gsp.reduction.graph_multiresolution(G, levels, sparsify=False)
    for i in range(1, levels + 1):
        np.testing.assert_array_equal(Gs[i].mr["idx"], z["mr_idx%d" % i])
        assert _rowwise(Gs[i].W.toarray(), csr_from(z, "mr_W%d" % i).toarray()) <= 1e-10
    for i in range(levels):
        assert _rowwise(Gs[i].mr["K_reg"].toarray(), csr_from(z, "mr_Kreg%d" % i).toarray()) <= 1e-10


@pytest.mark.parametrize("name", ["s256", "s1000", "grid"])
@pytest.mark.parametrize("dtype,tol", DTYPES)
def test_kron_reduction_goldens(gsp, golden, name, dtype, tol):
    z = golden("multiresolution")
    W = csr_from(z, name + "_W")
    ind = z[name + "_ind"]
    coords = np.random.default_rng(0).uniform(size=(W.shape[0], 2))
    G = gsp.graphs.Graph(W, coords=coords, dtype=dtype)
    Gk = gsp.reduction.kron_reduction(G, ind)
    assert Gk.dtype == G.dtype and Gk.N == ind.size
    np.testing.assert_array_equal(Gk.coords, coords[ind])
    got, want = Gk.W.toarray(), csr_from(z, name + "_kronW").toarray()
    assert _rowwise(got, want) <= tol
    assert _same_pattern(got, want)
    K = gsp.reduction.kron_reduction(laplacian(W) + 0.005 * sparse.eye(W.shape[0]), ind)
    assert sparse.isspmatrix_csr(K) and K.dtype == np.float64
    assert _rowwise(K.toarray(), csr_from(z, name + "_kreg").toarray()) <= 1e-10


def test_small_and_dense_paths_agree(gsp, golden, monkeypatch):
    z = golden("multiresolution")
    W = csr_from(z, "s1000_W")
    ind = z["s1000_ind"]
    M = laplacian(W) + 0.005 * sparse.eye(W.shape[0])
    small = gsp.reduction.kron_reduction(M, ind).toarray()
    monkeypatch.setattr(gsp.reduction, "SMALL_MAX", 0)
    dense = gsp.reduction.kron_reduction(M, ind).toarray()
    assert np.abs(small - dense).max() <= 1e-12 * np.abs(dense).max()
    # and both agree with the direct dense Schur complement
    assert np.abs(small - mro.kron_matrix(M, ind)).max() <= 1e-12 * np.abs(dense).max()


def test_removed_component_without_kept_neighbour(gsp):
    a = sparse.random(40, 40, density=0.15, random_state=1)
    a = a + a.T
    a.setdiag(0)
    b = sparse.csr_matrix(np.array([[0, 1.0, 0], [1.0, 0, 2.0], [0, 2.0, 0]]))
    W = sparse.block_diag([a, b]).tocsr()
    W.eliminate_zeros()
    ind = np.arange(0, 40, 2)                   # the 3-vertex component is removed entirely
    G = gsp.graphs.Graph(W, dtype=np.float64)
    got = gsp.reduction.kron_reduction(G, ind).W.toarray()
    assert np.all(np.isfinite(got))
    assert _rowwise(got, mro.kron_graph(a, ind)) <= 1e-10
    K = gsp.reduction.kron_reduction(laplacian(W), ind).toarray()
    assert np.all(np.isfinite(K))


def test_kron_reduction_errors(gsp):
    G = gsp.graphs.Sensor(100, seed=2, dtype=np.float64)
    G.compute_laplacian("normalized")
    with pytest.raises(NotImplementedError):
        gsp.reduction.kron_reduction(G, np.arange(50))
    D = sparse.random(30, 30, density=0.2, random_state=2, format="csr")
    with pytest.raises(NotImplementedError):
        gsp.reduction.kron_reduction(gsp.graphs.Graph(D, dtype=np.float64), np.arange(10))
    G = gsp.graphs.Sensor(100, seed=2, dtype=np.float64)
    with pytest.raises(NotImplementedError):
        gsp.reduction.graph_multiresolution(G, 1, downsampling_method="random")
    with pytest.raises(NotImplementedError):
        gsp.reduction.graph_multiresolution(G, 1, reduction_method="other")


def test_kron_reduction_matrix_errors(gsp, monkeypatch):
    """A non-symmetric matrix, and one whose removed block is not positive definite, raise
    ValueError -- through the one-CTA kernel and through the dense path."""
    W = gsp.graphs.Sensor(200, seed=3).W.to_scipy().astype(np.float64)
    L = laplacian(W)
    A = L.tolil()
    A[0, 1] += 0.25
    with pytest.raises(ValueError):
        gsp.reduction.kron_reduction(A.tocsr(), np.arange(0, 200, 2))
    ind = np.arange(0, 200, 2)
    with pytest.raises(ValueError):
        gsp.reduction.kron_reduction(-L, ind)
    monkeypatch.setattr(gsp.reduction, "SMALL_MAX", 0)
    with pytest.raises(ValueError):
        gsp.reduction.kron_reduction(-L, ind)


def test_explicit_zero_is_not_an_edge(gsp):
    """A stored zero between two components does not join them: resistances stay those of pinv,
    for the Laplacian given as a SciPy matrix and as a DeviceCSR (zeros removed on the device)."""
    import torch
    a = sparse.random(30, 30, density=0.2, random_state=4)
    a = a + a.T
    a.setdiag(0)
    a.eliminate_zeros()
    W = sparse.block_diag([a, a]).tocsr()
    C = laplacian(W).tocoo()
    L = sparse.csr_matrix((np.r_[C.data, 0.0, 0.0], (np.r_[C.row, 0, 45], np.r_[C.col, 45, 0])),
                          shape=C.shape)
    assert L.nnz == laplacian(W).nnz + 2            # the zeros are stored
    P = np.linalg.pinv(laplacian(W).toarray())
    d = np.diag(P)
    want = d[:, None] + d[None, :] - 2 * P
    Ld = gsp.graphs.DeviceCSR.from_scipy(L, torch.float64, torch.device("cuda"))
    assert int((Ld.data == 0).sum()) == 2
    for M in (L, Ld):
        got = gsp.utils.resistance_distance(M)
        assert np.abs(got - want).max() <= 1e-9 * np.abs(want).max()


def test_largest_eigenvector_chfsi_float32(gsp):
    """The float32 reflected ChFSI (tol 1e-5, float32 filter range) against ARPACK in float64
    on the same (float32-rounded) weights."""
    from scipy.sparse import linalg
    G = gsp.graphs.Sensor(5000, k=8, seed=4, order="morton")
    assert G.dtype == __import__("torch").float32
    v1 = G._largest_eigenvector(seed=3)
    np.testing.assert_array_equal(v1, G._largest_eigenvector(seed=3))
    L = G.L.to_scipy().astype(np.float64)
    v = v1 / np.linalg.norm(v1)
    theta = v @ (L @ v)
    upper = G._get_upper_bound()
    assert np.linalg.norm(L @ v - theta * v) <= 1e-4 * upper
    w = linalg.eigsh(L, 1, which="LA")[0][0]
    assert abs(theta - w) <= 1e-5 * w


def test_multiresolution_compute_full_eigen(gsp, golden):
    """compute_full_eigen=True: every level gets its full basis, and the split uses U[:, -1]."""
    z = golden("pyramid")
    levels = int(z["levels"])
    G = gsp.graphs.Graph(csr_from(z, "W0"), dtype=np.float64)
    Gs = gsp.reduction.graph_multiresolution(G, levels, sparsify=False, compute_full_eigen=True)
    for i, g in enumerate(Gs):
        assert len(g.e) == g.N and g._lmax_method == "fourier"
        if i:
            np.testing.assert_array_equal(g.mr["idx"], z["idx%d" % i])


def test_largest_eigenvector_chfsi(gsp):
    """Above the dense crossover the reflected ChFSI runs; seeded: same bits twice."""
    from scipy.sparse import linalg
    G = gsp.graphs.Sensor(5000, k=8, seed=4, dtype=np.float64, order="morton")
    v1 = G._largest_eigenvector(seed=3)
    v2 = G._largest_eigenvector(seed=3)
    np.testing.assert_array_equal(v1, v2)
    L = G.L.to_scipy().astype(np.float64)
    theta = v1 @ (L @ v1)
    assert np.linalg.norm(L @ v1 - theta * v1) <= 1e-10 * G._get_upper_bound() * 1.01
    w = linalg.eigsh(L, 1, which="LA")[0][0]
    assert abs(theta - w) <= 1e-9 * w


def test_resistance_distance_matches_pinv(gsp):
    a = sparse.random(80, 80, density=0.08, random_state=3)
    a = a + a.T
    a.setdiag(0)
    a.eliminate_zeros()
    disconnected = sparse.block_diag([a, sparse.csr_matrix(np.array([[0, 3.0], [3.0, 0]])),
                                      sparse.csr_matrix((1, 1))]).tocsr()
    for W in (gsp.graphs.Sensor(300, seed=5).W.to_scipy(), a, disconnected):
        L = laplacian(sparse.csr_matrix(W, dtype=np.float64)).toarray()
        P = np.linalg.pinv(L)
        d = np.diag(P)
        want = d[:, None] + d[None, :] - 2 * P
        got = gsp.utils.resistance_distance(gsp.graphs.Graph(W, dtype=np.float64))
        assert np.abs(got - want).max() <= 1e-9 * np.abs(want).max()
        got_m = gsp.utils.resistance_distance(sparse.csr_matrix(L))
        assert np.abs(got_m - want).max() <= 1e-9 * np.abs(want).max()
    G = gsp.graphs.Sensor(50, seed=1)
    G.compute_laplacian("normalized")
    with pytest.raises(ValueError):
        gsp.utils.resistance_distance(G)


@pytest.fixture(scope="module")
def sparsify_case(gsp):
    G = gsp.graphs.Sensor(3000, k=10, seed=6, dtype=np.float64, order="morton")
    eps = 0.3
    S1 = gsp.reduction.graph_sparsify(G, eps, seed=11)
    S2 = gsp.reduction.graph_sparsify(G, eps, seed=11)
    return G, eps, S1, S2


def test_graph_sparsify_properties(gsp, sparsify_case):
    G, eps, S1, S2 = sparsify_case
    import torch
    for a, b in ((S1.W.indptr, S2.W.indptr), (S1.W.indices, S2.W.indices),
                 (S1.W.data, S2.W.data)):
        assert torch.equal(a, b)
    assert S1.is_connected()
    assert not S1.is_directed()
    W, Ws = G.W.to_scipy().astype(np.float64), S1.W.to_scipy().astype(np.float64)
    assert (abs(Ws - Ws.T)).max() == 0
    assert ((Ws != 0).astype(int) - (W != 0).astype(int)).max() <= 0     # subset of the edges
    assert Ws.nnz < W.nnz
    np.testing.assert_array_equal(S1.coords, G.coords)

    # every weight is count * w / (q Pe) with integer counts summing to q
    N = G.N
    q = int(round(N * np.log(N) * 9 * (4 / 30.0) ** 2 / eps ** 2))
    R = gsp.utils.resistance_distance(G)
    T = sparse.tril(W, -1).tocoo()
    x = T.data * np.maximum(R[T.row, T.col], 0)
    Pe = x / x.sum()
    got = np.asarray(Ws[T.row, T.col]).ravel()
    counts = got * q * Pe / T.data
    assert np.abs(counts - np.round(counts)).max() <= 1e-4 * max(1.0, counts.max())
    counts = np.round(counts).astype(np.int64)
    assert counts.sum() == q

    # fixed-seed chi-square test of the counts against q Pe (bins of expected count >= 5)
    expected = q * Pe
    order = np.argsort(expected)
    e_sorted, c_sorted = expected[order], counts[order]
    groups = np.cumsum(e_sorted) // 5
    edges = np.flatnonzero(np.diff(groups)) + 1
    e_bins = np.add.reduceat(e_sorted, np.r_[0, edges])
    c_bins = np.add.reduceat(c_sorted, np.r_[0, edges])
    keep = e_bins >= 5
    chi2 = float((((c_bins - e_bins) ** 2) / e_bins)[keep].sum())
    dof = int(keep.sum()) - 1
    assert stats.chi2.sf(chi2, dof) > 1e-4, (chi2, dof)


def test_graph_sparsify_errors_and_matrix_branch(gsp, caplog):
    G = gsp.graphs.Sensor(1000, k=10, seed=8, dtype=np.float64)
    with pytest.raises(ValueError):
        gsp.reduction.graph_sparsify(G, 1.0)
    with pytest.raises(ValueError):
        gsp.reduction.graph_sparsify(G, 0.5 / np.sqrt(G.N))
    Gn = gsp.graphs.Sensor(1000, k=10, seed=8, dtype=np.float64)
    Gn.compute_laplacian("normalized")
    with pytest.raises(NotImplementedError):
        gsp.reduction.graph_sparsify(Gn, 0.5)
    L = G.L.to_scipy().astype(np.float64)
    Ls = gsp.reduction.graph_sparsify(L, 0.5, seed=2)
    assert sparse.isspmatrix_csr(Ls) and Ls.shape == L.shape
    assert np.abs(np.asarray(Ls.sum(axis=1))).max() <= 1e-9 * np.abs(Ls.diagonal()).max()
    assert abs(Ls - Ls.T).max() == 0
    # at the largest epsilon of the range q is about 1100 draws for about 5000 edges: the sample
    # leaves vertices isolated, and with maxiter=1 the reference's warning is logged
    S = gsp.reduction.graph_sparsify(gsp.graphs.Sensor(1000, k=10, seed=8, dtype=np.float64),
                                     0.999, maxiter=1, seed=1)
    assert not S.is_connected()
    assert "sparsified graph is disconnected" in caplog.text


def test_multiresolution_default_pipeline(gsp):
    """graph_multiresolution with its defaults (sparsify=True) on a 1e4-vertex k-NN graph:
    every level connected and undirected, the same seed gives bit-identical levels, and the
    pyramid on the sparsified levels reconstructs its input."""
    import time
    import torch
    G = gsp.graphs.Sensor(10_000, k=10, seed=1, order="morton")
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    Gs = gsp.reduction.graph_multiresolution(G, 3)
    torch.cuda.synchronize()
    elapsed = time.perf_counter() - t0
    print("graph_multiresolution(Sensor(1e4, k=10), 3): %.2f s, N = %s, nnz = %s"
          % (elapsed, [g.N for g in Gs], [g.W.nnz for g in Gs]))
    assert len(Gs) == 4
    for i, g in enumerate(Gs):
        assert g.is_connected()
        assert not g.is_directed()
        assert g.dtype == G.dtype
        if i:
            assert g.N < Gs[i - 1].N and g.mr["level"] == i - 1
            assert sparse.isspmatrix_csr(Gs[i - 1].mr["K_reg"])
            assert Gs[i - 1].mr["K_reg"].shape == (g.N, g.N)
    again = gsp.reduction.graph_multiresolution(
        gsp.graphs.Sensor(10_000, k=10, seed=1, order="morton"), 3)
    for g, h in zip(Gs, again):
        for a, b in ((g.W.indptr, h.W.indptr), (g.W.indices, h.W.indices),
                     (g.W.data, h.W.data)):
            assert torch.equal(a, b)
        np.testing.assert_array_equal(g.mr["idx"], h.mr["idx"])
    f = np.random.default_rng(0).standard_normal((G.N, 1))
    ca, pe = gsp.reduction.pyramid_analysis(Gs, f, order=30)
    rec, _ = gsp.reduction.pyramid_synthesis(Gs, ca[3], pe, order=30)
    assert np.linalg.norm(rec - f) / np.linalg.norm(f) <= 1e-5
