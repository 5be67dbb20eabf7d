"""Random graph models on the device (csrc/random_graphs.cu): bit-for-bit against the serial
restatement of oracle/random_graphs_oracle.py, independent of the launch shape, statistically
equal to the reference's own runs (tests/golden/random_graphs.npz), and at scale."""
import numpy as np
import pytest
from scipy import stats

from conftest import load_golden, relerr_cols
from oracle import pygsp_oracle as orc
from oracle import random_graphs_oracle as rgo

pytestmark = pytest.mark.gpu

F32_TOL = 1e-5          # the float32 filtering tolerance of tests/test_gpu_parity.py


@pytest.fixture(scope="module")
def gsp():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import pygsp_b200
    return pygsp_b200


@pytest.fixture(scope="module")
def golden():
    return load_golden("random_graphs")


@pytest.fixture
def rg(gsp):
    from pygsp_b200.graphs import random_graphs
    return random_graphs


def _case(g, name):
    z, M = g["sbm_%s_z" % name], g["sbm_%s_M" % name]
    directed, loops = (bool(f) for f in g["sbm_%s_flags" % name])
    return z, M, directed, loops


def _sbm(gsp, z, M, directed, loops, seed, **kw):
    return gsp.graphs.StochasticBlockModel(z.size, k=M.shape[0], z=z, M=M, directed=directed,
                                           self_loops=loops, seed=seed, backend="device", **kw)


def _key(seed):
    return int(np.random.default_rng(seed).integers(2 ** 63))


def _same_csr(W, ref):
    S = W.to_scipy()
    assert np.array_equal(S.indptr, ref.indptr)
    assert np.array_equal(S.indices, ref.indices)
    assert np.array_equal(S.data, ref.data)


SBM_CASES = ["default", "directed", "loops", "asym", "unsorted", "er"]


@pytest.mark.parametrize("name", SBM_CASES)
@pytest.mark.parametrize("target", [64, 1.0])
def test_sbm_matches_oracle(gsp, golden, rg, monkeypatch, name, target):
    monkeypatch.setattr(rg, "_CHUNK_TARGET", target)
    z, M, directed, loops = _case(golden, name)
    for seed in (0, 1, 2):
        G = _sbm(gsp, z, M, directed, loops, seed)
        ref, emitted = rgo.sbm_graph(z.size, M.shape[0], z, M, directed, loops, _key(seed),
                                     target)
        assert ref.nnz == emitted
        _same_csr(G.W, ref)


def test_erdos_renyi_matches_oracle(gsp):
    for directed, loops in ((False, False), (True, True)):
        G = gsp.graphs.ErdosRenyi(300, p=0.05, directed=directed, self_loops=loops, seed=11)
        ref, _ = rgo.sbm_graph(300, 1, np.zeros(300, int), np.array([[0.05]]), directed, loops,
                               _key(11))
        _same_csr(G.W, ref)
        assert G.is_directed() == directed


@pytest.mark.parametrize("N,m0,m", [(300, 1, 1), (500, 3, 2), (200, 5, 5), (64, 8, 3)])
def test_ba_matches_oracle(gsp, N, m0, m):
    for seed in (0, 5):
        G = gsp.graphs.BarabasiAlbert(N, m0=m0, m=m, seed=seed)
        _same_csr(G.W, rgo.ba_graph(N, m0, m, _key(seed)))


def test_launch_shape_and_repeat_independence(gsp, rg, monkeypatch):
    z = np.random.default_rng(3).integers(0, 4, 3000)
    M = np.full((4, 4), 0.002) + np.eye(4) * 0.01
    shapes = []
    for blocks in (0, 1, 0):
        monkeypatch.setattr(rg, "_MAX_BLOCKS", blocks)
        G = _sbm(gsp, z, M, False, False, 9)
        B = gsp.graphs.BarabasiAlbert(20000, m0=3, m=3, seed=9)
        shapes.append((G.W.to_scipy(), B.W.to_scipy(), B._rounds))
    for S, B, _ in shapes[1:]:
        assert (S != shapes[0][0]).nnz == 0 and (B != shapes[0][1]).nnz == 0
    assert shapes[0][2] >= 1


@pytest.mark.parametrize("name", SBM_CASES)
def test_sbm_statistics_match_reference(gsp, golden, name):
    z, M, directed, loops = _case(golden, name)
    ref = golden["sbm_%s_counts" % name]
    k = M.shape[0]
    ours = []
    for seed in range(300):
        G = _sbm(gsp, z, M, directed, loops, 10 ** 4 + seed)
        coo = G.W.to_scipy().tocoo()
        C = np.zeros((k, k), dtype=np.int64)
        np.add.at(C, (z[coo.row], z[coo.col]), 1)
        ours.append(C)
    ours = np.array(ours)
    se = np.sqrt(ours.var(0) / len(ours) + ref.var(0) / len(ref))
    assert (np.abs(ours.mean(0) - ref.mean(0)) / np.maximum(se, 1e-9)).max() < 4.5


@pytest.mark.parametrize("case", ["n300_m1", "n500_m2", "n1000_m4"])
def test_ba_degree_histogram_matches_reference(gsp, golden, case):
    N, m0, m = (int(v) for v in golden["ba_%s_params" % case])
    ref = golden["ba_%s_hist" % case]
    S = int(golden["ba_%s_nseeds" % case])
    ours = np.zeros(N, dtype=np.int64)
    for seed in range(S):
        deg = np.diff(gsp.graphs.BarabasiAlbert(N, m0=m0, m=m, seed=10 ** 5 + seed)
                      .W.to_scipy().indptr)
        ours += np.bincount(deg, minlength=N)[:N]
    # degrees 0 .. m + 7 one by one, then the tail
    cut = m + 8
    table = np.array([np.append(h[:cut], h[cut:].sum()) for h in (ours, ref)])
    table = table[:, table.sum(0) > 0]
    assert stats.chi2_contingency(table).pvalue > 1e-6


def test_structure(gsp):
    for loops in (False, True):
        G = gsp.graphs.StochasticBlockModel(2000, k=3, p=0.02, q=0.002, seed=4,
                                            self_loops=loops, backend="device")
        W = G.W.to_scipy()
        assert not G.is_directed() and (W != W.T).nnz == 0
        assert (W.diagonal().sum() > 0) == loops
        assert set(np.unique(W.data)) == {1.0}
    G = gsp.graphs.StochasticBlockModel(2000, k=3, p=0.02, q=0.002, seed=4, directed=True,
                                        backend="device", dtype=np.float64)
    assert G.is_directed() and str(G.W.dtype) == "torch.float64"
    assert G.W.to_scipy().diagonal().sum() == 0
    N, m0, m = 5000, 4, 3
    B = gsp.graphs.BarabasiAlbert(N, m0=m0, m=m, seed=1)
    _ba_structure(B, N, m0, m)


def _ba_structure(B, N, m0, m):
    import torch
    from pygsp_b200.graphs.csr import row_ids
    W = B.W
    assert W.nnz == 2 * m * (N - m0) and not B.is_directed()
    rows = row_ids(W.indptr)
    below = torch.bincount(rows[W.indices.long() < rows], minlength=N).cpu().numpy()
    assert (below[:m0] == 0).all() and (below[m0:] == m).all()
    assert bool((W.data == 1).all())


def test_connected(gsp):
    G = gsp.graphs.ErdosRenyi(400, p=0.02, connected=True, n_try=50, seed=2)
    assert G.is_connected()
    with pytest.raises(ValueError, match="could not be connected after 3 trials"):
        gsp.graphs.ErdosRenyi(50, p=0.0, connected=True, n_try=3, seed=1)
    with pytest.raises(ValueError, match="could not be connected after 2 trials"):
        gsp.graphs.StochasticBlockModel(60, k=2, p=0.5, q=0.0, connected=True, n_try=2, seed=1,
                                        backend="device")


def test_scale_ba_lmax_and_filter(gsp):
    import torch
    N, m0, m = 10 ** 6, 4, 4
    B = gsp.graphs.BarabasiAlbert(N, m0=m0, m=m, seed=0)
    _ba_structure(B, N, m0, m)
    W = B.W.to_scipy()
    dmax = int(np.diff(W.indptr).max())
    assert dmax > 500                       # hubs
    B.estimate_lmax()
    assert B.lmax >= dmax + 1
    x = np.random.default_rng(0).standard_normal((N, 4)).astype(np.float32)
    y = gsp.filters.Heat(B, 50).filter(x, order=30)
    L = orc.laplacian(W.astype(np.float64))
    ref = orc.filter_signal(L, B.lmax, orc.heat_kernels(B.lmax, 50), x.astype(np.float64),
                            order=30)
    assert relerr_cols(y, ref) <= F32_TOL
    S = gsp.graphs.StochasticBlockModel(10 ** 6, k=8, p=2e-5, q=2e-6, seed=0, backend="device")
    assert 0 < S.W.nnz < 2 ** 31 and not S.is_directed()
    del B, S
    torch.cuda.empty_cache()


def test_errors(gsp, rg, monkeypatch):
    with pytest.raises(ValueError, match="m cannot be above"):
        gsp.graphs.BarabasiAlbert(100, m0=2, m=3)
    for p in (-0.1, 1.5):
        with pytest.raises(ValueError, match="Probabilities"):
            gsp.graphs.ErdosRenyi(100, p=p)
    z = np.random.default_rng(0).permutation(np.repeat([0, 1], 20))
    M = np.array([[0.3, 0.1], [0.2, 0.3]])
    with pytest.raises(ValueError, match="asymmetric M"):
        gsp.graphs.StochasticBlockModel(40, k=2, z=z, M=M, backend="device")
    G = gsp.graphs.StochasticBlockModel(40, k=2, z=z, M=M, directed=True, backend="device")
    assert G.is_directed()
    called = []
    real = rg.nat.call
    monkeypatch.setattr(rg.nat, "call", lambda name, *a: (called.append(name), real(name, *a)))
    with pytest.raises(ValueError, match="at most 2"):
        gsp.graphs.ErdosRenyi(50000, p=1.0)
    assert called == ["gsp_sbm_count"]
