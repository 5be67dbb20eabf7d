"""Lanczos filtering on the CUDA engine (pygsp_b200/filters/approximations.py, csrc/krylov.cu)
against tests/golden/lanczos.npz, made by the unmodified PyGSP 0.6.1."""
import numpy as np
import pytest

from conftest import csr_from, load_golden

pytestmark = pytest.mark.gpu

GRAPHS = [str(g) for g in load_golden("lanczos")["graphs"]]
OP_GRAPHS = ("logo", "sensor")
DTYPES = [np.float32, np.float64]
# Normwise bounds on the fixtures.  float32: not measured on the device; a float32 run of the
# oracle (lanczos_oracle.lanczos_op(..., dtype=np.float32), all arithmetic in float32) is at most
# 1.3e-6 from the fixtures, and the engine sums in float64, so 1e-4 leaves a wide margin.
OP_BOUND = {np.float32: 1e-4, np.float64: 1e-9}


@pytest.fixture(scope="module")
def gsp():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import pygsp_b200
    return pygsp_b200


def kernels(z, g, name):
    """The fixture's filters, restated: Heat(scale=[5, 20]) on the reference's lmax, and the
    one-filter step kernel lambda x: (x <= 0.3 * lmax) * 1.0."""
    lmax = float(z[g + "_lmax"])
    if name == "heat":
        return [lambda x: np.exp(-5 * x / lmax), lambda x: np.exp(-20 * x / lmax)]
    return [lambda x: (x <= 0.3 * lmax) * 1.0]


def relnorm(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    nb = np.linalg.norm(b)
    return np.linalg.norm(a - b) / nb if nb > 0 else np.linalg.norm(a)


def _device(t):
    import torch
    return torch.device("cuda:%d" % torch.cuda.current_device())


@pytest.mark.parametrize("order", (1, 2, 20))
@pytest.mark.parametrize("g", GRAPHS)
def test_basis_against_reference(gsp, golden, g, order):
    import torch
    from pygsp_b200.graphs.csr import DeviceCSR
    z = golden("lanczos")
    L = csr_from(z, g + "_L")
    for A in (L, L.toarray(), DeviceCSR.from_scipy(L, torch.float64, _device(torch))):
        V, H, orth = gsp.filters.lanczos(A, order, z[g + "_x"])
        ref_V, ref_H = z["%s_V%d" % (g, order)], z["%s_H%d" % (g, order)]
        assert isinstance(V, np.ndarray) and V.shape == ref_V.shape and H.shape == ref_H.shape
        np.testing.assert_allclose(V, ref_V, rtol=1e-8, atol=1e-10)
        np.testing.assert_allclose(H, ref_H, rtol=1e-8, atol=1e-10 * np.abs(ref_H).max())
        np.testing.assert_allclose(orth, z["%s_orth%d" % (g, order)], rtol=1e-8, atol=1e-12)


def test_basis_of_several_signals(gsp, golden):
    """M > 1: independent processes, each signal's T in its block of H (the reference couples
    the processes and keeps the first T only)."""
    import torch
    from oracle import lanczos_oracle as lo
    z = golden("lanczos")
    L = csr_from(z, "sensor_L")
    x = np.random.default_rng(4).standard_normal((L.shape[0], 3))
    V, H, orth = gsp.filters.lanczos(L, 12, torch.as_tensor(x, device=_device(torch)))
    assert V.is_cuda and V.shape == (L.shape[0], 36) and H.shape == (12, 36)
    rV, rH, rorth = lo.lanczos(L, 12, x)
    np.testing.assert_allclose(V.cpu().numpy(), rV, rtol=1e-8, atol=1e-10)
    np.testing.assert_allclose(H, rH, rtol=1e-8, atol=1e-10 * np.abs(rH).max())
    np.testing.assert_allclose(orth, rorth, rtol=1e-8)


@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f64"])
@pytest.mark.parametrize("g", OP_GRAPHS)
def test_op_against_reference(gsp, golden, g, dtype):
    z = golden("lanczos")
    G = gsp.graphs.Graph(csr_from(z, g + "_W"), dtype=dtype)
    for fname in ("heat", "step"):
        f = gsp.filters.Filter(G, kernels(z, g, fname))
        for sig in ("s1", "s3"):
            key = "%s_%s_%s" % (g, fname, sig)
            for order in (1, 10, 30):
                y = gsp.filters.lanczos_op(f, z["%s_%s" % (g, sig)], order=order)
                ref = z["%s_o%d" % (key, order)]
                assert isinstance(y, np.ndarray) and y.shape == ref.shape and y.dtype == dtype
                assert relnorm(y, ref) <= OP_BOUND[dtype], (key, order)
            if fname == "heat":                       # approximation error of order 30
                assert relnorm(y, z[key + "_exact"]) <= max(1e-8, OP_BOUND[dtype])


@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f64"])
def test_breakdown(gsp, golden, dtype):
    z = golden("lanczos")
    G = gsp.graphs.Graph(csr_from(z, "logo_W"), dtype=dtype)
    f = gsp.filters.Filter(G, kernels(z, "logo", "heat"))
    tol = 1e-12 if dtype == np.float64 else 1e-6
    # a constant signal: L s = 0, beta_1 = 0 at once, the result is f(0) s = s for each filter
    s = np.full(G.N, 0.5)
    y = gsp.filters.lanczos_op(f, s, order=30)
    assert np.all(np.isfinite(y))
    np.testing.assert_allclose(y, np.concatenate([s, s]), rtol=0, atol=tol)
    # a zero column gives zeros, next to columns that do not
    S = np.random.default_rng(2).standard_normal((G.N, 3))
    S[:, 1] = 0
    y = gsp.filters.lanczos_op(f, S, order=20)
    assert np.all(np.isfinite(y)) and not y[:, 1].any()
    alone = gsp.filters.lanczos_op(f, S[:, 2], order=20)
    np.testing.assert_array_equal(y[:, 2], alone)


def test_eigenvector_response(gsp, golden):
    """An eigenvector u of Logo from the Fourier path: the response is f(lambda) u."""
    z = golden("lanczos")
    G = gsp.graphs.Graph(csr_from(z, "logo_W"), dtype=np.float64)
    G.compute_fourier_basis()
    f = gsp.filters.Filter(G, kernels(z, "logo", "heat"))
    for i in (0, 10, 500):
        u = np.ascontiguousarray(G.U[:, i])
        y = gsp.filters.lanczos_op(f, u, order=30)
        want = np.concatenate([k(max(G.e[i], 0.0)) * u for k in f._kernels])
        assert relnorm(y, want) <= 1e-9, i


def test_batch_independence(gsp):
    """A column's bits do not depend on the columns that share its batch, on chunking, or on
    the run."""
    import torch
    from pygsp_b200.filters.approximations import lanczos_op_device
    G = gsp.graphs.Sensor(20_000, k=10, seed=3, dtype=np.float32)
    f = gsp.filters.Heat(G, scale=[10, 40])
    gen = torch.Generator(device=G.device).manual_seed(0)
    X = torch.randn((G.N, 64), generator=gen, device=G.device, dtype=torch.float32)
    X[:, 7] = 0
    L = G.L
    y = lanczos_op_device(L, f.evaluate, X, 20)
    assert torch.isfinite(y).all() and not y[:, :, 7].any()
    assert torch.equal(y, lanczos_op_device(L, f.evaluate, X, 20))
    assert torch.equal(y, lanczos_op_device(L, f.evaluate, X, 20, max_columns=5))
    for j in (0, 31, 33, 63):
        alone = lanczos_op_device(L, f.evaluate, X[:, j:j + 1].contiguous(), 20)
        assert torch.equal(y[:, :, j:j + 1], alone), j


def test_kinds_shapes_and_errors(gsp, golden):
    import torch
    from scipy import sparse
    from pygsp_b200.graphs.csr import DeviceCSR
    z = golden("lanczos")
    W = csr_from(z, "sensor_W")
    G = gsp.graphs.Graph(W, dtype=np.float32)
    f = gsp.filters.Filter(G, kernels(z, "sensor", "heat"))
    s = z["sensor_s3"]
    ref = gsp.filters.lanczos_op(f, s, order=10)
    y = gsp.filters.lanczos_op(f, torch.as_tensor(s, dtype=torch.float32, device=G.device), 10)
    assert y.is_cuda and y.dtype == torch.float32 and tuple(y.shape) == (2 * G.N, 3)
    np.testing.assert_array_equal(y.cpu().numpy(), ref)
    y = gsp.filters.lanczos_op(f, torch.as_tensor(s[:, 0]), 10)
    assert torch.is_tensor(y) and not y.is_cuda and tuple(y.shape) == (2 * G.N,)
    np.testing.assert_array_equal(y.numpy(), gsp.filters.lanczos_op(f, s[:, 0], 10))

    # a stock graph and filter (SciPy L): float64 back, as cheby_op
    class StockGraph:
        N = G.N
        lmax = float(z["sensor_lmax"])
        L = (sparse.diags(np.asarray(W.sum(axis=1)).ravel()) - W).tocsr()

    class StockFilter:
        G = StockGraph()
        Nf = 2
        _kernels = kernels(z, "sensor", "heat")

        def evaluate(self, x):
            return np.array([k(x) for k in self._kernels])
    y = gsp.filters.lanczos_op(StockFilter(), s, order=10)
    assert isinstance(y, np.ndarray) and y.dtype == np.float64 and y.shape == (2 * G.N, 3)
    assert relnorm(y, z["sensor_heat_s3_o10"]) <= OP_BOUND[np.float32]

    with pytest.raises(ValueError):
        f.filter(s, method="lanczos")
    with pytest.raises(ValueError):
        gsp.filters.lanczos_op(f, s, order=0)
    with pytest.raises(ValueError):
        gsp.filters.lanczos(W, 0, s)
    with pytest.raises(ValueError, match="First dimension must be the number of vertices"):
        gsp.filters.lanczos_op(f, s[:-1], order=10)
    # a rectangular matrix is refused before any launch (the SpMM would read past the basis)
    R = DeviceCSR.from_scipy(sparse.random(G.N, 3 * G.N, 0.01, random_state=0, format="csr"),
                             torch.float32, G.device)
    with pytest.raises(ValueError, match="must be square"):
        gsp.filters.lanczos(R, 10, s)
    from pygsp_b200.filters.approximations import lanczos_op_device
    x = torch.as_tensor(s, dtype=torch.float32, device=G.device)
    with pytest.raises(ValueError, match="must be square"):
        lanczos_op_device(R, f.evaluate, x, 10)
    # no signal columns: empty results
    y = gsp.filters.lanczos_op(f, np.zeros((G.N, 0)), order=10)
    assert isinstance(y, np.ndarray) and y.shape == (2 * G.N, 0)
    V, H, orth = gsp.filters.lanczos(W, 5, np.zeros((G.N, 0)))
    assert V.shape == (G.N, 0) and H.shape == (5, 0) and orth.shape == (5,)


def test_wide_bank(gsp, golden):
    """18 filters: more than one pass of the combine over the basis (16 filters per pass), and an
    output of 18 blocks allocated before the columns are sized."""
    from oracle import lanczos_oracle as lo
    z = golden("lanczos")
    G = gsp.graphs.Graph(csr_from(z, "sensor_W"), dtype=np.float64)
    lmax = float(z["sensor_lmax"])
    bank = [(lambda t: (lambda x: np.exp(-t * x / lmax)))(t) for t in range(1, 19)]
    f = gsp.filters.Filter(G, bank)
    s = z["sensor_s3"]
    y = gsp.filters.lanczos_op(f, s, order=20)
    ref = lo.lanczos_op(f.evaluate, csr_from(z, "sensor_L"), s, order=20)
    assert y.shape == (18 * G.N, 3)
    assert relnorm(y, ref) <= 1e-9


@pytest.fixture(scope="module")
def config2(gsp):
    """BASELINE config 2: Sensor-type 2-D k-NN graph, 1e6 vertices, k = 10, Morton order."""
    G = gsp.graphs.Sensor(1_000_000, k=10, seed=0, order="morton", dtype=np.float32)
    yield G
    del G


def test_at_scale_against_chebyshev(gsp, config2, monkeypatch):
    """64 float32 signals, Heat(scale=50), order 30: Lanczos agrees with order-30 Chebyshev,
    and no vector of size N is copied to the host."""
    import torch
    from pygsp_b200.graphs.csr import DeviceCSR
    G = config2
    f = gsp.filters.Heat(G, scale=50)
    gen = torch.Generator(device=G.device).manual_seed(1)
    X = torch.randn((G.N, 64), generator=gen, device=G.device, dtype=torch.float32)
    cheb = gsp.filters.cheby_op(G, gsp.filters.compute_cheby_coeff(f, m=30), X)
    largest = []
    cpu = torch.Tensor.cpu

    def counted(self, *args, **kwargs):
        largest.append(self.numel())
        return cpu(self, *args, **kwargs)

    def leaves(self):
        raise AssertionError("the matrix left the device")
    monkeypatch.setattr(DeviceCSR, "to_scipy", leaves)
    monkeypatch.setattr(torch.Tensor, "cpu", counted)
    y = gsp.filters.lanczos_op(f, X, order=30)
    monkeypatch.undo()
    assert largest and max(largest) < G.N
    assert y.is_cuda and tuple(y.shape) == (G.N, 64)
    err = (torch.linalg.norm((y - cheb).double()) / torch.linalg.norm(cheb.double())).item()
    assert err <= 1e-4, err
