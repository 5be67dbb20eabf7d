"""Connectivity on the CUDA engine (pygsp_b200/graphs/connectivity.py, csrc/connectivity.cu)
against tests/golden/connectivity.npz, made by the unmodified PyGSP 0.6.1, and, at full size,
against scipy.sparse.csgraph on the host."""
import logging

import numpy as np
import pytest
from scipy import sparse
from scipy.sparse import csgraph

from conftest import csr_from, load_golden
from oracle import connectivity_oracle as co

pytestmark = pytest.mark.gpu

GRAPHS = [str(g) for g in load_golden("connectivity")["graphs"]]
SUBGRAPHS = [str(s) for s in load_golden("connectivity")["subgraphs"]]
DTYPES = [np.float32, np.float64]
MESSAGE = "Constructing subgraph for component of size {}."


@pytest.fixture(scope="module")
def gsp():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import pygsp_b200
    return pygsp_b200


def _launches(gsp):
    import ctypes
    lib = gsp._native.lib()
    lib.gsp_launch_count.restype = ctypes.c_uint64
    return int(lib.gsp_launch_count())


def _check_csr(W, ref, dtype):
    """W (DeviceCSR) equals the SciPy matrix ref: structure bit for bit, values after rounding
    to the graph's dtype."""
    assert W.shape == ref.shape
    np.testing.assert_array_equal(W.indptr.cpu().numpy(), ref.indptr)
    np.testing.assert_array_equal(W.indices.cpu().numpy(), ref.indices)
    got = W.data.cpu().numpy()
    assert got.dtype == dtype
    np.testing.assert_array_equal(got, ref.data.astype(dtype))


def _canonical(labels):
    """SciPy component labels -> the smallest vertex id of each component."""
    first = np.full(labels.max(initial=-1) + 1, labels.size)
    np.minimum.at(first, labels, np.arange(labels.size))
    return first[labels]


@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f64"])
@pytest.mark.parametrize("name", GRAPHS)
def test_against_reference(gsp, golden, caplog, name, dtype):
    z = golden("connectivity")
    G = gsp.graphs.Graph(csr_from(z, name + "_W"), lap_type="normalized", dtype=dtype)
    assert G.is_directed() == bool(z[name + "_directed"])
    assert G.is_connected() == bool(z[name + "_connected"])
    assert G.is_weighted() == bool(z[name + "_weighted"])
    if G.is_directed():
        with pytest.raises(NotImplementedError, match="Directed graphs not supported yet."):
            G.extract_components()
        return
    with caplog.at_level(logging.INFO):
        comps = G.extract_components()
    assert len(comps) == int(z[name + "_n_components"])
    sizes = [r.getMessage() for r in caplog.records if "Constructing subgraph" in r.getMessage()]
    assert sizes == [MESSAGE.format(C.N) for C in comps]
    for k, C in enumerate(comps):
        p = "%s_comp%d" % (name, k)
        assert type(C) is gsp.graphs.Graph
        ids = C.info["orig_idx"]
        assert isinstance(ids, np.ndarray) and ids.dtype == np.int64
        np.testing.assert_array_equal(ids, z[p + "_orig_idx"])
        _check_csr(C.W, csr_from(z, p + "_W"), dtype)
        assert C.lap_type == "normalized" and C.dtype == G.dtype and C.device == G.device
        assert C.L.shape == (C.N, C.N)


@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f64"])
@pytest.mark.parametrize("case", SUBGRAPHS)
def test_subgraph_against_reference(gsp, golden, case, dtype):
    import torch
    z = golden("connectivity")
    g = str(z[case + "_graph"])
    sel = z[case + "_sel"]
    G = gsp.graphs.Graph(csr_from(z, g + "_W"), coords=z[g + "_coords"],
                         plotting={"limits": [0, 1]}, dtype=dtype)
    G.set_signal(z[g + "_signal"], "sig")
    G.set_signal(torch.as_tensor(z[g + "_signal"], device=G.device), "sig_dev")
    ref = csr_from(z, case + "_W")
    selections = [sel, list(sel), torch.as_tensor(sel, device=G.device)]
    for s in selections:
        S = G.subgraph(s)
        assert type(S) is gsp.graphs.Graph and S.N == ref.shape[0]
        _check_csr(S.W, ref, dtype)
        assert S.lap_type == G.lap_type and S.plotting == G.plotting
        assert S.dtype == G.dtype and S.device == G.device
        np.testing.assert_array_equal(S.coords, z[case + "_coords"])
        assert isinstance(S.signals["sig"], np.ndarray)
        np.testing.assert_array_equal(S.signals["sig"], z[case + "_signal"])
        dev = S.signals["sig_dev"]
        assert torch.is_tensor(dev) and dev.device == G.device
        np.testing.assert_array_equal(dev.cpu().numpy(), z[case + "_signal"])


def test_doctests_and_errors(gsp, golden):
    z = golden("connectivity")
    G = gsp.graphs.Graph(csr_from(z, "doc_connected_W"), dtype=np.float64)
    np.testing.assert_array_equal(G.subgraph([0, 2, 1]).W.toarray(),
                                  [[0., 0., 3.], [0., 0., 4.], [3., 4., 0.]])
    assert G.is_connected()
    with pytest.raises(IndexError):
        G.subgraph([0, 4])
    with pytest.raises(IndexError):
        G.subgraph([-5])
    with pytest.raises(IndexError):
        G.subgraph(np.array([True, False, True]))
    with pytest.raises(IndexError):
        G.subgraph([0.5, 1.0])
    with pytest.raises(ValueError, match="G.N = 4"):
        G.set_signal(np.ones(3), "bad")
    G.set_signal(np.arange(4), "ids")
    np.testing.assert_array_equal(G.signals["ids"], np.arange(4))
    neg = gsp.graphs.Graph(csr_from(z, "negative_W"))
    assert neg.is_connected()
    assert [list(C.info["orig_idx"]) for C in neg.extract_components()] == [[0, 1], [2, 3]]
    E = gsp.graphs.Graph(np.zeros((0, 0)))
    with pytest.raises(IndexError):
        E.is_connected()
    assert E.extract_components() == []


def test_cache_launches_nothing(gsp, golden):
    z = golden("connectivity")
    for name in ("sensor", "random_loops"):
        G = gsp.graphs.Graph(csr_from(z, name + "_W"))
        first = G.is_connected()
        before = _launches(gsp)
        assert G.is_connected() is first
        assert _launches(gsp) == before


def test_stochastic_block_model(gsp):
    from pygsp_b200.graphs.generators import sbm_adjacency
    G = gsp.graphs.StochasticBlockModel(300, k=3, p=0.05, q=0.005, seed=4, connected=True)
    assert G.is_connected()
    with pytest.raises(ValueError, match="could not be connected after 3 trials"):
        gsp.graphs.StochasticBlockModel(50, k=2, p=0.0, q=0.0, seed=1, connected=True, n_try=3)
    for seed in (0, 7):
        G = gsp.graphs.StochasticBlockModel(2000, k=4, p=0.004, q=0.0004, seed=seed)
        W, zz = sbm_adjacency(2000, 4, None, 0.004, 0.0004, seed)
        assert (G.W.to_scipy() != W).nnz == 0
        np.testing.assert_array_equal(G.z, zz)


# ---------------------------------------------------------------------- full size
def _labels(G, positive_only=False):
    labels, n_components = G._component_labels(positive_only)
    return labels.cpu().numpy(), int(n_components.item())


def _scipy_labels(W):
    n, labels = csgraph.connected_components(W, directed=False)
    return _canonical(labels), n


@pytest.fixture(scope="module")
def config2(gsp):
    """BASELINE config 2: Sensor-type 2-D k-NN graph, 1e6 vertices, k = 10, Morton order."""
    G = gsp.graphs.Sensor(1_000_000, k=10, seed=0, order="morton", dtype=np.float32)
    yield G, G.W.to_scipy()
    del G


def test_full_size_labels(gsp, config2):
    G, W = config2
    ref, n = _scipy_labels(W)
    got, m = _labels(G)
    assert m == n and np.array_equal(got, ref)
    assert G.is_connected() == (n == 1)
    # a directed variant: W's structure with asymmetric weights, strongly connected iff W is
    Gd = gsp.graphs.Graph(W.multiply(1.0) + sparse.triu(W, k=1))
    n_strong, _ = csgraph.connected_components(Gd.W.to_scipy(), directed=True,
                                               connection="strong")
    assert Gd.is_directed() and Gd.is_connected() == (n_strong == 1)
    # the directed k-NN graph before symmetrisation
    from pygsp_b200.graphs.generators import knn_device
    nn, _ = knn_device(G.coords, 10)
    nn = nn.cpu().numpy()
    K = sparse.csr_matrix((np.ones(nn.size), nn.ravel(), np.arange(0, nn.size + 1, 10)),
                          shape=(G.N, G.N))
    K.sort_indices()
    n_strong, _ = csgraph.connected_components(K, directed=True, connection="strong")
    assert gsp.graphs.Graph(K).is_connected() == (n_strong == 1)


def test_percolated_grid(gsp):
    n1 = 1000
    N = n1 * n1
    right = np.ones(N - 1)
    right[n1 - 1::n1] = 0
    W = sparse.diags([right, np.ones(N - n1)], [1, n1], shape=(N, N), format="csr")
    W = (W + W.T).tocsr()
    keep = np.random.default_rng(5).random(N) >= 0.4
    D = sparse.diags(keep.astype(np.float64))
    W = (D @ W @ D).tocsr()
    W.eliminate_zeros()
    W.sort_indices()
    ref, n = _scipy_labels(W)
    assert n > 1000
    G = gsp.graphs.Graph(W)
    for positive_only in (False, True):
        got, m = _labels(G, positive_only)
        assert m == n and np.array_equal(got, ref)
    assert not G.is_connected()


def test_permuted_path_and_cycle(gsp):
    rng = np.random.default_rng(9)
    N = 2 ** 20
    perm = rng.permutation(N)
    a, b = perm[:-1], perm[1:]

    def sym(r, c, n):
        W = sparse.csr_matrix((np.ones(2 * r.size), (np.r_[r, c], np.r_[c, r])), shape=(n, n))
        W.sort_indices()
        return W
    G = gsp.graphs.Graph(sym(a, b, N))
    assert G.is_connected()
    assert _labels(G)[1] == 1
    cut = N // 3                                 # remove edge (perm[cut], perm[cut + 1])
    keep = np.arange(N - 1) != cut
    G = gsp.graphs.Graph(sym(a[keep], b[keep], N))
    assert not G.is_connected()
    got, m = _labels(G)
    want = np.empty(N, dtype=np.int64)
    want[perm[:cut + 1]] = perm[:cut + 1].min()
    want[perm[cut + 1:]] = perm[cut + 1:].min()
    assert m == 2 and np.array_equal(got, want)

    n = 100_000
    perm = rng.permutation(n)
    r, c = perm, np.roll(perm, -1)
    C = sparse.csr_matrix((np.ones(n), (r, c)), shape=(n, n))
    C.sort_indices()
    G = gsp.graphs.Graph(C)
    assert G.is_directed() and G.is_connected()
    C = sparse.csr_matrix((np.ones(n - 1), (r[1:], c[1:])), shape=(n, n))
    C.sort_indices()
    assert not gsp.graphs.Graph(C).is_connected()


def test_sbm_components(gsp):
    G = gsp.graphs.StochasticBlockModel(1_000_000, k=8, p=5e-5, q=5e-6, seed=3)
    W = G.W.to_scipy()
    ref, n = _scipy_labels(W)
    assert n > 1
    runs = [G.extract_components() for _ in range(2)]
    comps = runs[0]
    assert len(comps) == n
    roots = np.unique(ref)
    for C, root in zip(comps, roots):
        np.testing.assert_array_equal(C.info["orig_idx"], np.flatnonzero(ref == root))
        assert C.L.shape == (C.N, C.N)
    assert sum(C.N for C in comps) == G.N
    assert sum(C.W.nnz for C in comps) == G.W.nnz
    for A, B in zip(*runs):
        np.testing.assert_array_equal(A.info["orig_idx"], B.info["orig_idx"])
        for x, y in ((A.W.indptr, B.W.indptr), (A.W.indices, B.W.indices),
                     (A.W.data, B.W.data), (A.L.data, B.L.data)):
            assert bool((x == y).all())


def test_nothing_leaves_the_device(gsp, config2, monkeypatch):
    import torch
    from pygsp_b200.graphs.csr import DeviceCSR
    G, W = config2

    def leaves(self):
        raise AssertionError("the matrix left the device")
    monkeypatch.setattr(DeviceCSR, "to_scipy", leaves)
    G._connected = None
    connected = G.is_connected()
    comps = G.extract_components()
    half = np.random.default_rng(1).permutation(G.N)[:G.N // 2]
    S_sorted = G.subgraph(np.sort(half))
    S_shuffled = G.subgraph(torch.as_tensor(half, device=G.device))
    monkeypatch.undo()
    assert connected == (len(comps) == 1)
    assert S_sorted.W.nnz == S_shuffled.W.nnz
    ref = W[np.sort(half), :][:, np.sort(half)]
    _check_csr(S_sorted.W, ref.tocsr(), np.float32)
    ref = W[half, :][:, half].tocsr()
    ref.sort_indices()
    _check_csr(S_shuffled.W, ref, np.float32)
