"""Differential operator on the CUDA engine (pygsp_b200/graphs/difference.py,
csrc/difference.cu) against tests/golden/difference.npz, made by the unmodified PyGSP 0.6.1,
and, at full size, against the identities it must satisfy on the 1e6-vertex config-2 graph."""
import logging

import numpy as np
import pytest
from scipy import sparse

from conftest import csr_from, load_golden, relerr_cols
from oracle import pygsp_oracle as orc

pytestmark = pytest.mark.gpu

GRAPHS = [str(g) for g in load_golden("difference")["graphs"]]
LAP_TYPES = ("combinatorial", "normalized")
# (dtype, D values, grad / div outputs, energy)
DTYPES = [(np.float64, 1e-12, 1e-12, 1e-10), (np.float32, 2e-6, 1e-5, 1e-5)]


@pytest.fixture(scope="module")
def gsp():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import pygsp_b200
    return pygsp_b200


def _graph(gsp, z, name, dtype, lap_type="combinatorial"):
    G = gsp.graphs.Graph(csr_from(z, name + "_W"), dtype=dtype)
    G.compute_laplacian(lap_type)
    return G


def _ref_D(z, name, lap_type):
    p = "%s_%s_" % (name, lap_type)
    shape = (int(z[name + "_W_shape"][0]), int(z[name + "_n_edges"]))
    return sparse.csc_matrix((z[p + "D_data"], z[p + "D_indices"], z[p + "D_indptr"]), shape=shape)


def _max_abs(M):
    """max |M| of a small sparse matrix (0 when it has no entries)."""
    return float(np.abs(M.toarray()).max(initial=0))


def _close_cols(got, ref, tol, M, x):
    """relerr_cols(got, ref) <= tol for M x.  A column that is exactly zero in the reference
    (terms that cancel exactly: SciPy rounds each product, the kernel contracts to FMA) is
    held to tol * (|M| |x|) entry by entry instead."""
    got = np.asarray(got)
    assert got.shape == ref.shape
    if not ref.size:
        return
    g, r = got.reshape(len(ref), -1), ref.reshape(len(ref), -1)
    x = np.abs(x)
    bound = abs(M) @ (x[:, None] if x.ndim == 1 else x)
    zero = np.abs(r).max(axis=0) == 0
    if np.any(~zero):
        assert relerr_cols(g[:, ~zero], r[:, ~zero]) <= tol
    assert np.all(np.abs(g[:, zero]) <= tol * bound[:, zero])


@pytest.mark.parametrize("dtype,tol_d,tol_p,tol_e", DTYPES)
@pytest.mark.parametrize("lap_type", LAP_TYPES)
@pytest.mark.parametrize("name", GRAPHS)
def test_against_reference(gsp, golden, name, lap_type, dtype, tol_d, tol_p, tol_e):
    z = golden("difference")
    p = "%s_%s_" % (name, lap_type)
    G = _graph(gsp, z, name, dtype, lap_type)
    assert G.n_edges == int(z[name + "_n_edges"]) == G.Ne
    s, t, w = G.get_edge_list()
    assert s.dtype == np.int32 and t.dtype == np.int32 and w.dtype == dtype
    np.testing.assert_array_equal(s, z[name + "_sources"])
    np.testing.assert_array_equal(t, z[name + "_targets"])
    np.testing.assert_array_equal(w, z[name + "_weights"].astype(dtype))

    G.compute_differential_operator()
    D, ref = G.D, _ref_D(z, name, lap_type)
    assert D.shape == ref.shape and D.T.shape == ref.shape[::-1] and D.nnz == D.T.nnz == ref.nnz
    # structure: D^T is the reference's CSC, D its tocsr(), bit for bit
    np.testing.assert_array_equal(D.T.indptr.cpu().numpy(), ref.indptr)
    np.testing.assert_array_equal(D.T.indices.cpu().numpy(), ref.indices)
    ref_csr = ref.tocsr()
    np.testing.assert_array_equal(D.indptr.cpu().numpy(), ref_csr.indptr)
    np.testing.assert_array_equal(D.indices.cpu().numpy(), ref_csr.indices)
    for got, want in ((D.T.data, ref.data), (D.data, ref_csr.data)):
        got = got.cpu().numpy().astype(np.float64)
        assert np.all(np.abs(got - want) <= tol_d * np.abs(want))
    csc = D.to_scipy_csc()
    assert sparse.isspmatrix_csc(csc) and _max_abs(csc - ref) <= tol_d * _max_abs(ref)

    for v in ("x", "X"):
        x = z[name + "_" + v]
        _close_cols(G.grad(x), z[p + "grad_" + v], tol_p, ref.T, x)
    for v in ("y", "Y"):
        y = z[name + "_" + v]
        _close_cols(G.div(y), z[p + "div_" + v], tol_p, ref, y)

    L = orc.laplacian(csr_from(z, name + "_W"), lap_type)
    for key, x in (("energy_x", z[name + "_x"]), ("energy_X", z[name + "_X"])):
        e = G.dirichlet_energy(x)
        assert e.dtype == np.float64 and np.shape(e) == np.shape(z[p + key])
        scale = np.abs(x).T @ np.abs(L) @ np.abs(x)        # no cancellation in the bound
        assert np.all(np.abs(e - z[p + key]) <= tol_e * np.maximum(scale, 1e-300))


@pytest.mark.parametrize("lap_type", LAP_TYPES)
@pytest.mark.parametrize("name", ["tri_undirected", "tri_directed", "path4", "path4_directed",
                                  "logo", "er_directed", "small_directed", "random_loops"])
def test_D_Dt_is_the_laplacian(gsp, golden, name, lap_type):
    z = golden("difference")
    G = _graph(gsp, z, name, np.float64, lap_type)
    G.compute_differential_operator()
    D, Dt, L = G.D.to_scipy(), G.D.T.to_scipy(), G.L.to_scipy()
    assert _max_abs(D.T - Dt) == 0
    assert _max_abs(D @ Dt - L) <= 1e-12 * max(_max_abs(L), 1)


def test_doctest_values(gsp, golden):
    """difference.py:94-130, 216-322 and graph.py:680-698, 997-1015."""
    z = golden("difference")

    def op(name, lap="combinatorial"):
        G = _graph(gsp, z, name, np.float64, lap)
        G.compute_differential_operator()
        return G

    np.testing.assert_allclose(op("tri_undirected").D.toarray(),
                               [[-1.41421356, 0], [1.41421356, -1], [0, 1]], atol=1e-8)
    np.testing.assert_allclose(op("tri_undirected", "normalized").D.toarray(),
                               [[-1, 0], [0.81649658, -0.57735027], [0, 1]], atol=1e-8)
    np.testing.assert_allclose(op("tri_directed").D.toarray(),
                               [[-1, 1, 0], [1, -1, -0.70710678], [0, 0, 0.70710678]], atol=1e-8)
    np.testing.assert_allclose(op("tri_directed", "normalized").D.toarray(),
                               [[-0.70710678, 0.70710678, 0],
                                [0.63245553, -0.63245553, -0.4472136], [0, 0, 1]], atol=1e-8)
    printed = {("path4", "combinatorial"): ("[ 2.  2. -2.]", "[-2.  4. -2.  0.]"),
               ("path4_directed", "combinatorial"):
                   ("[ 1.41421356  1.41421356 -1.41421356]",
                    "[-1.41421356  2.82842712 -1.41421356  0.        ]"),
               ("path4", "normalized"):
                   ("[ 1.41421356  1.41421356 -0.82842712]",
                    "[-2.          2.82842712 -1.41421356  0.        ]"),
               ("path4_directed", "normalized"):
                   ("[ 1.41421356  1.41421356 -0.82842712]",
                    "[-2.          2.82842712 -1.41421356  0.        ]")}
    for (name, lap), (g, d) in printed.items():
        G = op(name, lap)
        assert str(G.grad([0, 2, 4, 2])) == g
        assert str(G.div([2, -2, 0])) == d
    for name, energy, grad in (("path5", 8.0, "[2. 0. 2. 0.]"),
                               ("path5_directed", 4.0, "[1.41421356 0.         1.41421356 0.        ]")):
        G = _graph(gsp, z, name, np.float64)
        assert G.dirichlet_energy([0, 2, 2, 4, 4]) == energy
        G.compute_differential_operator()
        assert str(G.grad([0, 2, 2, 4, 4])) == grad
    s, t, w = _graph(gsp, z, "edges_directed", np.float64).get_edge_list()
    assert (list(s), list(t), list(w)) == ([0, 1, 1], [1, 0, 2], [3, 3, 4])
    s, t, w = _graph(gsp, z, "edges_undirected", np.float64).get_edge_list()
    assert (list(s), list(t), list(w)) == ([0, 1], [1, 2], [3, 4])
    # the reference's Logo doctest (difference.py:134-140), through D.T.dot / D.dot
    G = _graph(gsp, z, "logo", np.float64)
    G.compute_differential_operator()
    s = np.random.default_rng().normal(size=G.N)
    assert np.linalg.norm(G.D.dot(G.D.T.dot(s)) - G.L.dot(s)) < 1e-10


def test_empty_graphs(gsp, golden):
    z = golden("difference")
    for lap in LAP_TYPES:
        G = _graph(gsp, z, "zeros", np.float64, lap)
        assert G.n_edges == 0 and G.D.shape == (11, 0) and G.D.nnz == 0 and G.D.T.shape == (0, 11)
        assert G.grad(np.ones(11)).shape == (0,)
        np.testing.assert_array_equal(G.div(np.zeros(0)), np.zeros(11))
        np.testing.assert_array_equal(G.div(np.zeros((0, 2))), np.zeros((11, 2)))
        H = _graph(gsp, z, "identity", np.float64, lap)
        assert H.n_edges == 11 and H.D.shape == (11, 11) and H.D.nnz == 0
        np.testing.assert_array_equal(H.grad(np.arange(11.0)), np.zeros(11))
        np.testing.assert_array_equal(H.div(np.arange(11.0)), np.zeros(11))
        assert len(H.get_edge_list()[0]) == 11


def test_cache_rules_and_errors(gsp, golden, caplog):
    z = golden("difference")
    G = _graph(gsp, z, "sensor", np.float64)
    assert G._D is None
    G.compute_differential_operator()
    D = G.D
    assert G.D is D
    G.compute_laplacian("combinatorial")                     # same type: kept
    assert G.D is D
    G.compute_laplacian("normalized")
    assert G._D is None
    with caplog.at_level(logging.WARNING):
        D = G.D
    assert "call G.compute_differential_operator() once beforehand" in caplog.text
    ref = _ref_D(z, "sensor", "normalized")
    assert _max_abs(D.to_scipy_csc() - ref) <= 1e-12
    with pytest.raises(ValueError, match="G.Ne = {}".format(G.Ne)):
        G.div(np.ones(G.Ne + 1))
    with pytest.raises(ValueError, match="G.N = "):
        G.grad(np.ones(G.N + 1))
    with pytest.raises(ValueError, match="G.N = "):
        G.dirichlet_energy(np.ones(G.N - 1))
    G.n_edges = 2 ** 30 + G._n_loops                           # nnz(D) = 2^31: refused
    with pytest.raises(ValueError, match="2\\^31"):
        G.compute_differential_operator()


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_lists_tensors_blocks(gsp, golden, dtype):
    import torch
    z = golden("difference")
    G = _graph(gsp, z, "random_loops", dtype)
    G.compute_differential_operator()
    rng = np.random.default_rng(3)
    X = rng.standard_normal((G.N, 3))
    Y = rng.standard_normal((G.Ne, 3))
    X0, Y0 = X.copy(), Y.copy()
    gX, dY, eX = G.grad(X), G.div(Y), G.dirichlet_energy(X)
    np.testing.assert_array_equal(X, X0)
    np.testing.assert_array_equal(Y, Y0)
    assert gX.dtype == dtype and gX.shape == (G.Ne, 3) and dY.shape == (G.N, 3)
    assert eX.dtype == np.float64 and eX.shape == (3, 3)
    tol = 1e-6 if dtype == np.float32 else 1e-15
    for j in range(3):
        np.testing.assert_allclose(G.grad(list(X[:, j])), gX[:, j], rtol=tol, atol=tol)
        np.testing.assert_allclose(G.div(Y[:, j]), dY[:, j], rtol=tol, atol=tol)
        assert G.dirichlet_energy(X[:, j]) == pytest.approx(eX[j, j], rel=1e-5 if
                                                            dtype == np.float32 else 1e-12)
    Xt = torch.as_tensor(X, device=G.device)
    Yt = torch.as_tensor(Y, device=G.device)
    gt, dt, et = G.grad(Xt), G.div(Yt), G.dirichlet_energy(Xt[:, 0])
    assert torch.is_tensor(gt) and gt.is_cuda and gt.dtype == G.dtype
    assert torch.is_tensor(dt) and dt.is_cuda and torch.is_tensor(et) and et.dim() == 0
    np.testing.assert_allclose(gt.cpu().numpy(), gX, rtol=tol, atol=tol)
    np.testing.assert_allclose(dt.cpu().numpy(), dY, rtol=tol, atol=tol)
    np.testing.assert_array_equal(Xt.cpu().numpy(), X0)


# ---------------------------------------------------------------------- full size
@pytest.fixture(scope="module", params=[np.float32, np.float64], ids=["f32", "f64"])
def config2(gsp, request):
    """BASELINE config 2: Sensor-type 2-D k-NN graph, 1e6 vertices, k = 10, Morton order."""
    G = gsp.graphs.Sensor(1_000_000, k=10, seed=0, order="morton", dtype=request.param)
    yield G
    del G


def test_full_size_identities(gsp, config2, monkeypatch):
    import torch
    from pygsp_b200.graphs.csr import DeviceCSR
    G = config2
    f64 = G.dtype == torch.float64

    def leaves(self):
        raise AssertionError("the matrix left the device")
    monkeypatch.setattr(DeviceCSR, "to_scipy", leaves)
    gen = torch.Generator(device=G.device).manual_seed(11)
    X = torch.randn((G.N, 4), generator=gen, device=G.device, dtype=G.dtype)
    Y = torch.randn((G.Ne, 4), generator=gen, device=G.device, dtype=G.dtype)
    G.compute_differential_operator()
    D = G.D
    assert D.shape == (G.N, G.Ne) and D.nnz == 2 * (G.Ne - G._n_loops)
    gX, dY, E = G.grad(X), G.div(Y), G.dirichlet_energy(X)
    g1, d1 = G.grad(X[:, 0]), G.div(Y[:, 0])
    LX = G.L.dot(X)
    monkeypatch.undo()

    # div(grad x) = L x
    assert relerr_cols(G.div(gX).cpu().numpy(), LX.cpu().numpy()) <= (1e-12 if f64 else 1e-5)
    assert relerr_cols(g1.cpu().numpy(), gX[:, 0].cpu().numpy()) <= (1e-15 if f64 else 1e-6)
    assert relerr_cols(d1.cpu().numpy(), dY[:, 0].cpu().numpy()) <= (1e-15 if f64 else 1e-6)
    # adjointness <grad x, y> = <x, div y> and energy = |grad x|^2
    lhs = (gX.double() * Y.double()).sum(0)
    rhs = (X.double() * dY.double()).sum(0)
    scale = (gX.double().abs() * Y.double().abs()).sum(0)
    assert torch.all((lhs - rhs).abs() <= (1e-10 if f64 else 1e-5) * scale)
    sq = (gX.double() ** 2).sum(0)
    assert torch.all((torch.diagonal(E) - sq).abs() <= (1e-10 if f64 else 1e-5) * sq)
    # grad of a constant: zero up to the rounding of c * D[i, k]
    c = 3.7
    gc = G.grad(torch.full((G.N,), c, device=G.device, dtype=G.dtype))
    assert float(gc.abs().max()) <= 1e-6 * c * float(D.data.abs().max())
    # determinism: a second build and second products are bit-identical
    G.compute_differential_operator()
    D2 = G.D
    for a, b in ((D.indptr, D2.indptr), (D.indices, D2.indices), (D.data, D2.data),
                 (D.T.indptr, D2.T.indptr), (D.T.indices, D2.T.indices), (D.T.data, D2.T.data)):
        assert torch.equal(a, b)
    assert torch.equal(G.grad(X), gX) and torch.equal(G.div(Y), dY)
