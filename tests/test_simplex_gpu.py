"""Simplex-constrained Tikhonov classification on the CUDA engine (pygsp_b200/learning.py,
csrc/simplex.cu) against tests/golden/simplex.npz -- the unmodified PyGSP 0.6.1 run with the
pyunlocbox stand-in -- and against oracle/learning_oracle.py for shapes without a fixture."""
import numpy as np
import pytest

from conftest import csr_from, load_golden
from oracle import learning_oracle as lo

pytestmark = pytest.mark.gpu

CASES = [str(c) for c in load_golden("simplex")["cases"]]
F64, F32 = np.float64, np.float32


@pytest.fixture(scope="module")
def gsp():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import pygsp_b200
    return pygsp_b200


def graph(gsp, z, c, dtype):
    G = gsp.graphs.Graph(csr_from(z, c + "_W"), dtype=dtype)
    G._lmax, G._lmax_method = float(z[c + "_lmax"]), "lanczos"
    return G


def relmax(a, b):
    return np.abs(np.asarray(a, dtype=np.float64) - b).max() / max(np.abs(b).max(), 1e-300)


def run(gsp, z, c, dtype, **kw):
    G = graph(gsp, z, c, dtype)
    kw.setdefault("verbosity", "NONE")
    return gsp.learning.classification_tikhonov_simplex(G, z[c + "_y"], z[c + "_M"],
                                                        tau=float(z[c + "_tau"]), **kw)


@pytest.mark.parametrize("c", CASES)
def test_default_stop_float64(gsp, golden, c):
    z = golden("simplex")
    X = run(gsp, z, c, F64)
    rec = gsp.learning.last_solve
    assert isinstance(X, np.ndarray) and X.dtype == np.float64 and X.shape == z[c + "_sol"].shape
    assert rec["niter"] == int(z[c + "_niter"]) and rec["crit"] == str(z[c + "_crit"])
    assert relmax(X, z[c + "_sol"]) <= 1e-10
    assert relmax(rec["objective"], z[c + "_obj"]) <= 1e-10


@pytest.mark.parametrize("c", CASES)
def test_default_stop_float32(gsp, golden, c):
    z = golden("simplex")
    X = run(gsp, z, c, F32)
    ref = z[c + "_sol"]
    assert X.dtype == np.float32
    assert relmax(X, ref) <= 1e-4
    assert np.all(X >= 0) and np.abs(X.astype(np.float64).sum(axis=1) - 1).max() <= 1e-5
    assert np.mean(X.argmax(axis=1) == ref.argmax(axis=1)) >= 0.99


@pytest.mark.parametrize("k", (1, 2, 17))
@pytest.mark.parametrize("c", CASES)
def test_fixed_iteration_counts(gsp, golden, c, k):
    z = golden("simplex")
    for dtype, tol in ((F64, 1e-10), (F32, 1e-5)):
        X = run(gsp, z, c, dtype, rtol=None, maxit=k)
        assert gsp.learning.last_solve["niter"] == k
        assert gsp.learning.last_solve["crit"] == "MAXIT"
        assert relmax(X, z["%s_sol%d" % (c, k)]) <= tol


# on the ring fixture these fire at iterations 13, 10, 46, 78, 23 and 1 (oracle), each with a
# margin of a few per cent on its threshold
STOPS = [dict(atol=0.1, rtol=None), dict(dtol=1e-2, rtol=None), dict(rtol=2e-2), dict(xtol=2e-3, rtol=None),
         dict(maxit=23, rtol=None), dict(maxit=0, rtol=None)]


@pytest.mark.parametrize("batch", (16, 5))
@pytest.mark.parametrize("stop", STOPS, ids=lambda s: "-".join("%s=%s" % kv for kv in s.items()))
def test_each_stopping_rule(gsp, golden, monkeypatch, stop, batch):
    """Every rule fires at the oracle's iteration, and the iterate returned is the one at the
    stop even when the batch enqueued runs past it (batch 16 never divides the stops)."""
    monkeypatch.setattr(gsp.learning, "SIMPLEX_BATCH", batch)
    z = golden("simplex")
    c = "ring"
    ref, niter, crit, obj = lo.solve(csr_from(z, c + "_L"), z[c + "_y"], z[c + "_M"],
                                     float(z[c + "_tau"]), float(z[c + "_lmax"]), **stop)
    X = run(gsp, z, c, F64, **stop)
    rec = gsp.learning.last_solve
    assert (rec["niter"], rec["crit"]) == (niter, crit)
    if batch == 16 and niter > 1:
        assert (niter + 1) % batch != 0                      # the stop falls inside a batch
    assert relmax(X, ref) <= 1e-10
    assert relmax(rec["objective"], obj) <= 1e-10


def sensor_problem(gsp, C, dtype):
    G = gsp.graphs.Sensor(300, seed=3, dtype=dtype)
    G.estimate_lmax()
    rng = np.random.default_rng(C)
    y = rng.integers(0, C, G.N).astype(float)
    y[0] = C - 1                                              # C classes exactly
    M = rng.uniform(size=G.N) > 0.5
    M[0] = True
    return G, y, M


@pytest.mark.parametrize("C", (1, 2, 3, 31, 32, 33, 64, 256))
def test_class_counts_against_the_oracle(gsp, C):
    for dtype, tol in ((F64, 1e-10), (F32, 1e-4)):
        G, y, M = sensor_problem(gsp, C, dtype)
        X = gsp.learning.classification_tikhonov_simplex(G, y, M, tau=0.5, verbosity="NONE")
        rec = gsp.learning.last_solve
        ref, niter, crit, _ = lo.solve(G.L.to_scipy().astype(np.float64), y, M, 0.5, G.lmax)
        assert X.shape == (G.N, C)
        if dtype == F64:
            assert (rec["niter"], rec["crit"]) == (niter, crit)
            assert relmax(X, ref) <= tol
        else:
            X17 = gsp.learning.classification_tikhonov_simplex(G, y, M, tau=0.5, rtol=None,
                                                               maxit=17)
            ref17, _, _, _ = lo.solve(G.L.to_scipy().astype(np.float64), y, M, 0.5, G.lmax,
                                      rtol=None, maxit=17)
            assert relmax(X17, ref17) <= tol
        assert np.all(X >= 0) and np.abs(X.astype(np.float64).sum(axis=1) - 1).max() <= 1e-5
    y[5] = C                                                  # C + 1 classes
    if C == 256:
        with pytest.raises(ValueError, match="256"):
            gsp.learning.classification_tikhonov_simplex(G, y, M)


def test_input_handling(gsp, golden):
    import torch
    z = golden("simplex")
    c = "sensor"
    G = graph(gsp, z, c, F64)
    y, M = z[c + "_y"].copy(), z[c + "_M"].copy()
    assert np.isnan(y[~M]).all()
    y0, M0 = y.copy(), M.copy()
    X = gsp.learning.classification_tikhonov_simplex(G, y, M, tau=0.1, verbosity="NONE")
    np.testing.assert_array_equal(y, y0)
    np.testing.assert_array_equal(M, M0)
    y2 = y.copy()
    y2[~M] = 123.0                                            # ignored off the mask
    np.testing.assert_array_equal(
        gsp.learning.classification_tikhonov_simplex(G, y2, M, verbosity="NONE"), X)
    yt = torch.as_tensor(y, device=G.device)
    Xt = gsp.learning.classification_tikhonov_simplex(G, yt, torch.as_tensor(M), verbosity="NONE")
    assert torch.is_tensor(Xt) and Xt.device == G.device and Xt.dtype == torch.float64
    np.testing.assert_array_equal(Xt.cpu().numpy(), X)
    assert torch.isnan(yt[torch.as_tensor(~M, device=G.device)]).all()
    with pytest.raises(ValueError, match="Tau"):
        gsp.learning.classification_tikhonov_simplex(G, y, M, tau=0)
    with pytest.raises(ValueError, match="Tau"):
        gsp.learning.classification_tikhonov_simplex(G, y, M, tau=-1.0)
    with pytest.raises(ValueError):
        gsp.learning.classification_tikhonov_simplex(G, y, M[:-1])
    y3 = y.copy()
    y3[np.flatnonzero(M)[0]] = -1
    with pytest.raises(ValueError, match="non-negative"):
        gsp.learning.classification_tikhonov_simplex(G, y3, M)
    with pytest.raises(TypeError):
        gsp.learning.classification_tikhonov_simplex(G, y, M, step=0.1)
    with pytest.raises(ValueError):
        gsp.learning.classification_tikhonov_simplex(G, y, M, verbosity="LOUD")


def test_scale_sensor_1m(gsp):
    import torch
    G = gsp.graphs.Sensor(1_000_000, k=10, seed=1, order="morton")
    G.estimate_lmax()
    rng = np.random.default_rng(0)
    coords = np.asarray(G.coords)
    y = (np.floor(coords[:, 0] * 5) + 5 * (coords[:, 1] > 0.5)).clip(0, 9)
    M = rng.uniform(size=G.N) < 0.05
    y[~M] = np.nan
    X = gsp.learning.classification_tikhonov_simplex(G, y, M, tau=1.0, verbosity="NONE")
    rec = gsp.learning.last_solve
    assert X.shape == (G.N, 10) and X.dtype == np.float32
    assert np.all(X >= 0) and np.abs(X.astype(np.float64).sum(axis=1) - 1).max() <= 1e-5
    assert rec["objective"][-1] < rec["objective"][0]
    X2 = gsp.learning.classification_tikhonov_simplex(G, y, M, tau=1.0, verbosity="NONE")
    np.testing.assert_array_equal(X, X2)                       # order-fixed reductions
    np.testing.assert_array_equal(rec["objective"], gsp.learning.last_solve["objective"])
    # projected-gradient residual after 2000 iterations, in float64 on the host
    Xc = gsp.learning.classification_tikhonov_simplex(G, y, M, tau=1.0, rtol=None, maxit=2000,
                                                      verbosity="NONE").astype(np.float64)
    lab, _ = lo.labels_of(y, M)
    L = G.L.to_scipy().astype(np.float64)
    res = lo.residual(L, Xc, lab, 1.0, G.lmax)
    assert res <= 1e-3 * np.linalg.norm(Xc)
    del Xc
    torch.cuda.empty_cache()
