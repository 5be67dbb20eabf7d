"""Graph total-variation prox on the CUDA engine (pygsp_b200/optimization.py, csrc/tv.cu) against
oracle/optimization_oracle.py: the iteration itself at fixed counts, converged runs against the
exact prox through the duality-gap certificate, the stop rule, column independence, the A / At
path and the errors."""
import ctypes

import numpy as np
import pytest

import tv_graphs as tg
from oracle import difference_oracle as do
from oracle import optimization_oracle as oo

pytestmark = pytest.mark.gpu

F64, F32 = np.float64, np.float32
CU_MEMPOOL_ATTR_USED_MEM_CURRENT = 7          # cuda.h, enum CUmemPool_attribute


@pytest.fixture(scope="module")
def gsp():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import pygsp_b200
    return pygsp_b200


def make(gsp, W, dtype=F64, lap="combinatorial"):
    """Device graph and oracle D; both use lmax of the oracle's D D^T."""
    G = gsp.graphs.Graph(W, lap_type=lap, dtype=dtype)
    D = do.differential_operator(W, lap)
    if D.shape[1]:
        G._lmax, G._lmax_method = tg.lmax_of(D), "lanczos"
    G.compute_differential_operator()
    return G, D


def signal(G, nsig=3, seed=0):
    return np.random.default_rng(seed).normal(size=(G.N, nsig))


CASES = {
    "weighted": lambda: (tg.geometric(), "combinatorial"),
    "directed": lambda: (tg.directed(), "combinatorial"),
    "normalized": lambda: (tg.geometric(50, 5), "normalized"),
    "disconnected": lambda: (tg.disconnected(), "combinatorial"),
    "loops": lambda: (tg.with_loops(), "combinatorial"),
}


@pytest.mark.parametrize("maxit", [1, 2, 10, 50])
@pytest.mark.parametrize("case", sorted(CASES))
def test_iteration_matches_oracle_float64(gsp, case, maxit):
    W, lap = CASES[case]()
    G, D = make(gsp, W, F64, lap)
    x = signal(G)
    z = gsp.optimization.prox_tv(x, 0.3, G, tol=0, maxit=maxit)
    rec = gsp.optimization.last_solve
    ref = oo.prox_tv_fgp(x, 0.3, D, G.lmax, tol=0, maxit=maxit)
    assert z.shape == x.shape and z.dtype == np.float64
    assert (rec["niter"], rec["crit"]) == (maxit, "MAXIT")
    assert np.abs(z - ref["z"]).max() <= oo.F64_Z * np.abs(x).max()
    for key in ("objective", "gap"):
        assert rec[key].shape == ref[key].shape
        assert np.abs(rec[key] - ref[key]).max() <= oo.F64_HIST * np.abs(ref[key]).max()


def converged(gsp, G, x, gamma, D):
    z = gsp.optimization.prox_tv(x, gamma, G, tol=1e-12, maxit=4000)
    gap = gsp.optimization.last_solve["gap"][-1]
    zs = oo.prox_tv_exact(x, gamma, D)
    assert gap >= 0
    assert np.linalg.norm(z - zs.reshape(z.shape)) <= np.sqrt(2 * gap) + 1e-10 * np.abs(x).max()
    return z, zs


SOLVED = {
    "sensor": lambda gsp: (gsp.graphs.Sensor(200, seed=3, dtype=F64).W.to_scipy(), "combinatorial"),
    "grid": lambda gsp: (tg.grid(), "combinatorial"),
    "six_decades": lambda gsp: (tg.six_decades(), "combinatorial"),
    "directed": lambda gsp: (tg.directed(), "combinatorial"),
    "normalized": lambda gsp: (tg.geometric(50, 5), "normalized"),
    "disconnected": lambda gsp: (tg.disconnected(), "combinatorial"),
    "loops": lambda gsp: (tg.with_loops(), "combinatorial"),
}


@pytest.mark.parametrize("case", sorted(SOLVED))
def test_converged_against_exact(gsp, case):
    W, lap = SOLVED[case](gsp)
    G, D = make(gsp, W, F64, lap)
    converged(gsp, G, signal(G, 2, seed=1), 0.4, D)


@pytest.mark.parametrize("gamma", [0.1, 0.7, 3.0])
def test_path_against_tv1d(gsp, gamma):
    G, D = make(gsp, tg.path(64))
    y = 2 * np.random.default_rng(4).normal(size=64)
    z, _ = converged(gsp, G, y, gamma, D)
    gap = gsp.optimization.last_solve["gap"][-1]
    assert np.linalg.norm(z - oo.tv1d_exact(y, gamma)) <= np.sqrt(2 * gap) + 1e-10


def test_sensor_1000_gap_bounds_distance(gsp):
    """Too many edges for BVLS: a run to a much smaller gap stands in for z*, and the two
    certificates bound the distance between the runs."""
    G = gsp.graphs.Sensor(1000, seed=0, dtype=F64)
    x = signal(G, 1, seed=2)[:, 0]
    z = gsp.optimization.prox_tv(x, 0.5, G)
    assert isinstance(z, np.ndarray) and z.shape == x.shape
    gap = gsp.optimization.last_solve["gap"][-1]
    z_ref = gsp.optimization.prox_tv(x, 0.5, G, tol=0, maxit=3000)
    gap_ref = gsp.optimization.last_solve["gap"][-1]
    assert 0 <= gap_ref < gap
    assert np.linalg.norm(z - z_ref) <= np.sqrt(2 * gap) + np.sqrt(2 * gap_ref)


@pytest.mark.parametrize("case", ["weighted", "directed", "loops"])
def test_float32_against_float64(gsp, case):
    W, lap = CASES[case]()
    x = signal(make(gsp, W)[0])
    z64 = gsp.optimization.prox_tv(x, 0.3, make(gsp, W, F64, lap)[0], tol=0, maxit=50)
    z32 = gsp.optimization.prox_tv(x, 0.3, make(gsp, W, F32, lap)[0], tol=0, maxit=50)
    assert z32.dtype == np.float32
    assert np.abs(z32 - z64).max() <= oo.F32_Z * np.abs(x).max()


@pytest.mark.parametrize("dtype", [F64, F32])
@pytest.mark.parametrize("nsig", [1, 3, 64, 300])
def test_columns_are_independent_and_runs_reproducible(gsp, nsig, dtype):
    G, _ = make(gsp, tg.geometric(), dtype)
    x = signal(G, nsig, seed=nsig)
    z = gsp.optimization.prox_tv(x, 0.3, G, tol=0, maxit=20)
    np.testing.assert_array_equal(gsp.optimization.prox_tv(x, 0.3, G, tol=0, maxit=20), z)
    for j in sorted({0, nsig // 2, nsig - 1}):
        zj = gsp.optimization.prox_tv(x[:, j], 0.3, G, tol=0, maxit=20)
        np.testing.assert_array_equal(zj, z[:, j])


# gammas where the oracle's stop is not within 1e-9 (relative) of the threshold
@pytest.mark.parametrize("case,gamma", [("weighted", 0.3), ("directed", 0.2), ("normalized", 0.5),
                                        ("disconnected", 1.0)])
def test_stop_matches_oracle_and_returns_the_stopping_iterate(gsp, case, gamma):
    W, lap = CASES[case]()
    G, D = make(gsp, W, F64, lap)
    x = signal(G)
    tol = 1e-3
    ref = oo.prox_tv_fgp(x, gamma, D, G.lmax, tol=tol)
    P = ref["objective"]
    for k in range(1, ref["niter"] + 1):                    # no test is a near tie
        rel = abs(P[k] - P[k - 1]) / abs(P[k])
        assert abs(rel - tol) > 1e-9 * tol
    z = gsp.optimization.prox_tv(x, gamma, G, tol=tol)
    rec = gsp.optimization.last_solve
    assert (rec["niter"], rec["crit"]) == (ref["niter"], ref["crit"]) and rec["crit"] == "RTOL"
    z_fixed = gsp.optimization.prox_tv(x, gamma, G, tol=0, maxit=rec["niter"])
    np.testing.assert_array_equal(z, z_fixed)
    assert np.abs(z - ref["z"]).max() <= oo.F64_Z * np.abs(x).max()


def test_stop_later_than_one_batch(gsp):
    G, D = make(gsp, tg.six_decades())
    x = signal(G, 1)
    z = gsp.optimization.prox_tv(x, 0.3, G, tol=1e-6, maxit=500)
    k = gsp.optimization.last_solve["niter"]
    assert k > gsp.optimization.TV_BATCH
    np.testing.assert_array_equal(z, gsp.optimization.prox_tv(x, 0.3, G, tol=0, maxit=k))


@pytest.mark.parametrize("dtype", [F64, F32])
def test_trivial_cases(gsp, dtype):
    import torch
    G, _ = make(gsp, tg.geometric(), dtype)
    c = np.full((G.N, 2), 1.25)
    z = gsp.optimization.prox_tv(c, 0.3, G)
    assert (gsp.optimization.last_solve["niter"], gsp.optimization.last_solve["crit"]) == (1, "RTOL")
    np.testing.assert_array_equal(z, c.astype(dtype))
    x = signal(G)
    for kw in (dict(gamma=0), dict(gamma=0.3, maxit=0)):
        z = gsp.optimization.prox_tv(x, G=G, **kw)
        assert gsp.optimization.last_solve["niter"] == 0
        np.testing.assert_array_equal(z, x.astype(dtype))
    E = gsp.graphs.Graph(np.zeros((5, 5)), dtype=dtype)
    xe = torch.arange(5, dtype=torch.float64, device="cuda")
    ze = gsp.optimization.prox_tv(xe, 0.3, E)
    assert torch.is_tensor(ze) and ze.is_cuda and ze.dtype == E.dtype
    assert torch.equal(ze.double(), xe) and gsp.optimization.last_solve["niter"] == 0
    assert ze.data_ptr() != xe.data_ptr()


def test_large_gamma_gives_component_means(gsp):
    W = tg.disconnected()
    G, D = make(gsp, W)
    x = signal(G, 2)
    gamma = 2 * tg.mean_bound(W, D, x)
    z = gsp.optimization.prox_tv(x, gamma, G, tol=1e-12, maxit=4000)
    gap = gsp.optimization.last_solve["gap"][-1]
    assert np.linalg.norm(z - tg.component_means(W, x)) <= np.sqrt(2 * gap) + 1e-10


def test_cuda_tensor_in_and_out_input_untouched(gsp):
    import torch
    G, _ = make(gsp, tg.geometric())
    x = torch.as_tensor(signal(G), device="cuda")
    keep = x.clone()
    z = gsp.optimization.prox_tv(x, 0.3, G, tol=0, maxit=5)
    assert torch.is_tensor(z) and z.shape == x.shape and torch.equal(x, keep)
    np.testing.assert_array_equal(z.cpu().numpy(),
                                  gsp.optimization.prox_tv(keep.cpu().numpy(), 0.3, G, tol=0, maxit=5))


def test_a_identity_matches_fused_path(gsp):
    G, _ = make(gsp, tg.geometric())
    x = signal(G)
    z = gsp.optimization.prox_tv(x, 0.3, G, tol=0, maxit=40)
    za = gsp.optimization.prox_tv(x, 0.3, G, A=lambda v: v, At=lambda v: v, tol=0, maxit=40)
    assert np.abs(za - z).max() <= oo.F64_Z * np.abs(x).max()


def test_a_scaled_identity_is_gamma_times_s(gsp):
    G, _ = make(gsp, tg.geometric())
    x = signal(G)
    s = 1.7
    za = gsp.optimization.prox_tv(x, 0.2, G, A=lambda v: s * v, At=lambda v: s * v, nu=s * s,
                                  tol=0, maxit=40)
    z = gsp.optimization.prox_tv(x, 0.2 * s, G, tol=0, maxit=40)
    assert np.abs(za - z).max() <= oo.F64_Z * np.abs(x).max()


def test_a_diagonal_against_oracle(gsp):
    import torch
    G, D = make(gsp, tg.geometric())
    x = signal(G, 2)
    d = np.random.default_rng(9).uniform(0.5, 1.5, G.N)
    dt = torch.as_tensor(d, device="cuda")[:, None]
    nu = float(d.max() ** 2)
    z = gsp.optimization.prox_tv(x, 0.3, G, A=lambda v: dt * v, At=lambda v: dt * v, nu=nu,
                                 tol=0, maxit=30)
    rec = gsp.optimization.last_solve
    ref = oo.prox_tv_fgp(x, 0.3, D, G.lmax, A=lambda v: d[:, None] * v,
                         At=lambda v: d[:, None] * v, nu=nu, tol=0, maxit=30)
    assert np.abs(z - ref["z"]).max() <= oo.F64_Z * np.abs(x).max()
    assert np.abs(rec["gap"] - ref["gap"]).max() <= oo.F64_HIST * np.abs(ref["gap"]).max()


def test_errors(gsp):
    G, _ = make(gsp, tg.geometric())
    x = signal(G)
    prox = gsp.optimization.prox_tv
    for kw in (dict(gamma=-1), dict(gamma=0.3, nu=0), dict(gamma=0.3, tol=-1e-3),
               dict(gamma=0.3, maxit=-1), dict(gamma=0.3, A=lambda v: v)):
        with pytest.raises(ValueError):
            prox(x, G=G, **kw)
    bad = x.copy()
    bad[3, 1] = np.nan
    with pytest.raises(ValueError):
        prox(bad, 0.3, G)
    with pytest.raises(ValueError, match="First dimension"):
        prox(x[:-1], 0.3, G)
    with pytest.raises(TypeError):
        prox(x, 0.3, G, A=lambda v: v.cpu().numpy(), At=lambda v: v)
    with pytest.raises(TypeError):
        prox(x, 0.3, G, A=lambda v: v, At=lambda v: v[:-1])


@pytest.fixture(scope="module")
def pool_used(gsp):
    """Bytes in use in the current device's default memory pool, after a synchronise."""
    import torch
    if torch.cuda.get_allocator_backend() == "cudaMallocAsync":
        pytest.skip("torch's own blocks would share the default memory pool")
    torch.zeros(1, device="cuda")                           # the primary context exists
    cuda = ctypes.CDLL("libcuda.so.1")
    dev = ctypes.c_int()
    assert cuda.cuDeviceGet(ctypes.byref(dev), torch.cuda.current_device()) == 0
    pool = ctypes.c_void_p()
    assert cuda.cuDeviceGetDefaultMemPool(ctypes.byref(pool), dev) == 0

    def used():
        torch.cuda.synchronize()
        value = ctypes.c_uint64()
        assert cuda.cuMemPoolGetAttribute(pool, CU_MEMPOOL_ATTR_USED_MEM_CURRENT,
                                          ctypes.byref(value)) == 0
        return value.value
    return used


def test_device_pool_released(gsp, pool_used):
    from pygsp_b200 import _native as nat
    G, _ = make(gsp, tg.geometric())
    x = signal(G)
    before = pool_used()
    gsp.optimization.prox_tv(x, 0.3, G)
    gsp.optimization.prox_tv(x, 0.3, G, A=lambda v: v, At=lambda v: v, maxit=5)
    assert pool_used() == before
    with pytest.raises(nat.NativeError, match="bad iteration range"):
        import torch
        z = torch.empty(G.N * 3, dtype=torch.float64, device="cuda")
        scal = torch.zeros(nat.FISTA_HISTORY + 2, dtype=torch.float64, device="cuda")
        D = G.D
        nat.call("gsp_prox_tv_f64", nat.i64(G.N), nat.i64(G.Ne), nat.i64(D.nnz), D.indptr,
                 D.indices, D.data, D.T.indptr, D.T.indices, D.T.data, z, nat.i64(3),
                 nat.f64(0.3), nat.f64(0.1), nat.f64(0), nat.i32(5), z, z, z, nat.i32(0),
                 nat.i32(2), nat.i32(1), scal, nat.stream_ptr())
    assert pool_used() == before
