"""graph_sparsify(resistances='sketch') on the device (pygsp_b200/reduction.py _edge_resistances,
csrc/resistance.cu): the sketch kernels and the CG solves against the dense restatement with the
same signs (oracle/resistance_sketch_oracle.py), the estimates against exact resistances, the
sparsifier's properties, the errors, and a graph past the dense factor's limit."""
import time

import numpy as np
import pytest
from scipy import sparse, stats

from oracle import resistance_sketch_oracle as rso

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gsp():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import pygsp_b200
    return pygsp_b200


def _edges(gsp, G):
    """(Ld, start, end, weights) as graph_sparsify forms them."""
    from pygsp_b200.graphs.csr import row_ids
    red = gsp.reduction
    Ld = red._device_matrix(G.L, G.device)
    rows, cols = row_ids(Ld.indptr), Ld.indices.long()
    w = -Ld.data
    edge = (rows > cols) & (w >= 1e-10)
    return Ld, rows[edge], cols[edge], w[edge]


def _host_w(G):
    return G.W.to_scipy().astype(np.float64).tocsr()


CASES = {
    "grid12": (lambda g: g.graphs.Grid2d(12, dtype=np.float64), 769),
    "sensor500": (lambda g: g.graphs.Sensor(500, k=10, seed=2, dtype=np.float64), 769),
    "two_components": (lambda g: g.graphs.Graph(rso.two_component_graph(), dtype=np.float64), 769),
    "partial_block": (lambda g: g.graphs.Grid2d(12, dtype=np.float64), 300),
    "float32": (lambda g: g.graphs.Sensor(500, k=10, seed=2, dtype=np.float32), 769),
}


def test_sketch_kernel_matches_oracle(gsp):
    """gsp_jl_sketch_f64 writes D^-1/2 B^T W^1/2 Q^T / sqrt(k) with the oracle's signs, for blocks
    that start inside a word, inside a Philox block, and span three Philox blocks."""
    import torch
    from pygsp_b200 import _native as nat
    G = gsp.graphs.Sensor(500, k=10, seed=2, dtype=np.float64)
    W = _host_w(G)
    Ld, _, _, _ = _edges(gsp, G)
    dinv = torch.as_tensor(rso._dinv(W), device=G.device)
    key, k = 0x5EED, 700
    for j0, width in ((0, 256), (8, 8), (120, 256), (256, 44), (696, 4)):
        Y = torch.full((G.N, width), np.nan, dtype=torch.float64, device=G.device)
        nat.call("gsp_jl_sketch_f64", nat.i64(G.N), Ld.indptr, Ld.indices, Ld.data, dinv,
                 nat.u64(key), nat.i64(j0), nat.i64(width), nat.i64(k), Y, nat.stream_ptr())
        want = rso.sketch_rhs(W, key, k, j0, width)
        got = Y.cpu().numpy()
        assert np.abs(got - want).max() <= 1e-13 * np.abs(want).max(), (j0, width)


@pytest.mark.parametrize("name", sorted(CASES))
def test_device_equals_oracle(gsp, name):
    """_edge_resistances against the dense pinv solve with the same key and k, per edge to
    relative 1e-5.  Measured on an H100 80GB HBM3: at most 8.7e-8 (the two-component graph, whose
    13-vertex CG runs past convergence until its stall rule stops it) and 2.2e-10 elsewhere."""
    make, k = CASES[name]
    G = make(gsp)
    seed = 5
    Ld, start, end, _ = _edges(gsp, G)
    R = gsp.reduction._edge_resistances(Ld, start, end, k, seed).cpu().numpy()
    s, e, want = rso.sketch_resistances(_host_w(G), gsp.reduction._sampling_seed(seed, 1 << 20), k)
    np.testing.assert_array_equal(start.cpu().numpy(), s)
    np.testing.assert_array_equal(end.cpu().numpy(), e)
    rel = float(np.abs(R / want - 1).max())
    print("%s: max relative difference %.2e" % (name, rel))
    assert rel <= 1e-5


@pytest.fixture(scope="module")
def sensor3000(gsp):
    G = gsp.graphs.Sensor(3000, k=10, seed=6, dtype=np.float64, order="morton")
    Ld, start, end, w = _edges(gsp, G)
    k = gsp.reduction._sketch_dim(G.N)
    R = gsp.reduction._edge_resistances(Ld, start, end, k, 11)
    return G, start, end, w, R


def test_accuracy_against_exact(gsp, sensor3000):
    G, start, end, w, R = sensor3000
    s, e = start.cpu().numpy(), end.cpu().numpy()
    Rx = gsp.utils.resistance_distance(G)[s, e]
    ratio = np.abs(R.cpu().numpy() / Rx - 1)
    print("max %.3f median %.4f" % (ratio.max(), np.median(ratio)))
    assert ratio.max() <= 0.5
    assert np.median(ratio) <= 0.06
    foster = float((w * R).sum())
    assert abs(foster / (G.N - 1) - 1) <= 0.01


def test_sparsifier_properties(gsp, sensor3000):
    import torch
    G, start, end, w, R = sensor3000
    eps = 0.3
    S1 = gsp.reduction.graph_sparsify(G, eps, seed=11, resistances="sketch")
    S2 = gsp.reduction.graph_sparsify(G, eps, seed=11, resistances="sketch")
    for a, b in ((S1.W.indptr, S2.W.indptr), (S1.W.indices, S2.W.indices),
                 (S1.W.data, S2.W.data)):
        assert torch.equal(a, b)
    assert S1.is_connected()
    assert not S1.is_directed()
    W, Ws = _host_w(G), _host_w(S1)
    assert (abs(Ws - Ws.T)).max() == 0
    assert ((Ws != 0).astype(int) - (W != 0).astype(int)).max() <= 0     # subset of the edges
    assert Ws.nnz < W.nnz
    np.testing.assert_array_equal(S1.coords, G.coords)

    # P~_e exactly as sampled: w_e R~_e rounded to 32 bits relative to its largest value
    N = G.N
    q = int(round(N * np.log(N) * 9 * (4 / 30.0) ** 2 / eps ** 2))
    x = (w * torch.clamp(R, min=0))
    kq = torch.round(x / x.max() * 2.0 ** 32).to(torch.int64)
    Pe = (kq.double() / int(kq.sum().item())).cpu().numpy()
    s, e, wh = (x.cpu().numpy().copy() for x in (start, end, w))
    got = np.asarray(Ws[s, e]).ravel()
    counts = got * q * Pe / wh
    assert np.abs(counts - np.round(counts)).max() <= 1e-4 * max(1.0, counts.max())
    counts = np.round(counts).astype(np.int64)
    assert counts.sum() == q

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

    # the quadratic forms: x^T L_s x / x^T L x averages to 1 (E[L_s] = L for any P~ > 0)
    L = sparse.csgraph.laplacian(W)
    Ls = sparse.csgraph.laplacian(Ws)
    X = np.random.default_rng(0).standard_normal((N, 64))
    ratio = np.einsum("ij,ij->j", X, Ls @ X) / np.einsum("ij,ij->j", X, L @ X)
    assert abs(ratio.mean() - 1) <= 0.1


def test_matrix_branch(gsp):
    G = gsp.graphs.Sensor(1000, k=10, seed=8, dtype=np.float64)
    L = G.L.to_scipy().astype(np.float64)
    assert np.abs(np.asarray(L.sum(axis=1))).max() <= 1e-12 * L.diagonal().max()
    assert abs(L - L.T).max() == 0
    Ls = gsp.reduction.graph_sparsify(L, 0.5, seed=2, resistances="sketch")
    assert sparse.isspmatrix_csr(Ls) and Ls.shape == L.shape
    assert np.abs(np.asarray(Ls.sum(axis=1))).max() <= 1e-9 * np.abs(Ls.diagonal()).max()
    assert abs(Ls - Ls.T).max() == 0
    assert ((Ls != 0).astype(int) - (L != 0).astype(int)).max() <= 0
    Ls2 = gsp.reduction.graph_sparsify(L, 0.5, seed=2, resistances="sketch")
    assert (Ls != Ls2).nnz == 0


def test_errors(gsp):
    G = gsp.graphs.Sensor(200, k=6, seed=3, dtype=np.float64)
    with pytest.raises(ValueError, match="resistances"):
        gsp.reduction.graph_sparsify(G, 0.5, resistances="dense")
    with pytest.raises(ValueError, match="sketch_dim"):
        gsp.reduction.graph_sparsify(G, 0.5, resistances="sketch", sketch_dim=0)
    L = G.L.to_scipy().astype(np.float64).tolil()
    L[0, 1] -= 0.25                                    # asymmetric
    with pytest.raises(ValueError, match="symmetric"):
        gsp.reduction.graph_sparsify(L.tocsr(), 0.5, resistances="sketch")
    L = G.L.to_scipy().astype(np.float64).tolil()
    j = next(c for c in L.rows[0] if c != 0)
    L[0, j] = L[j, 0] = 0.5                            # a negative weight
    with pytest.raises(ValueError, match="non-negative"):
        gsp.reduction.graph_sparsify(L.tocsr(), 0.5, resistances="sketch")
    Gn = gsp.graphs.Sensor(200, k=6, seed=3, dtype=np.float64)
    Gn.compute_laplacian("normalized")
    with pytest.raises(NotImplementedError):
        gsp.reduction.graph_sparsify(Gn, 0.5, resistances="sketch")


def test_past_the_dense_limit(gsp):
    import torch
    free, _ = torch.cuda.mem_get_info()
    if free < 16 * 2 ** 30:
        pytest.skip("needs 16 GB of free device memory")
    G = gsp.graphs.Sensor(100_000, k=10, seed=1, order="morton")
    with pytest.raises(ValueError, match="dense factor"):
        gsp.reduction.graph_sparsify(G, 0.3, seed=3)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    S = gsp.reduction.graph_sparsify(G, 0.3, seed=3, resistances="sketch")
    torch.cuda.synchronize()
    print("graph_sparsify(Sensor(1e5), 0.3, resistances='sketch'): %.2f s"
          % (time.perf_counter() - t0))
    assert S.is_connected()
    assert not S.is_directed()
    assert S.W.nnz < G.W.nnz
    Ld, start, end, w = _edges(gsp, G)
    R = gsp.reduction._edge_resistances(Ld, start, end, gsp.reduction._sketch_dim(G.N), 3)
    assert abs(float((w * R).sum()) / (G.N - 1) - 1) <= 0.01
