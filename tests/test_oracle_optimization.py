"""The total-variation prox oracle (oracle/optimization_oracle.py) checked against itself and
against independent solutions: the exact 1-D denoiser on paths, the box-constrained dual by
BVLS, the duality-gap certificate along the iteration, the component-mean solution at large
gamma, the stop-rule edge cases, and the drift behind the device tests' tolerances."""
import numpy as np
import pytest
from scipy import sparse

import tv_graphs as tg
from oracle import difference_oracle as do
from oracle import optimization_oracle as oo

RNG = np.random.default_rng(0)


def op(W, lap="combinatorial"):
    D = do.differential_operator(W, lap)
    return D, tg.lmax_of(D)


GRAPHS = {
    "weighted": lambda: op(tg.geometric()),
    "directed": lambda: op(tg.directed()),
    "normalized": lambda: op(tg.geometric(50, 5), "normalized"),
    "disconnected": lambda: op(tg.disconnected()),
}


@pytest.mark.parametrize("gamma", [0.0, 0.05, 0.3, 1.0, 4.0])
@pytest.mark.parametrize("n", [2, 17, 60])
def test_exact_dual_matches_tv1d_on_paths(n, gamma):
    y = np.random.default_rng(n).normal(size=n) * 2
    D = do.differential_operator(tg.path(n))
    z = oo.prox_tv_exact(y, gamma, D)[:, 0]
    np.testing.assert_allclose(z, oo.tv1d_exact(y, gamma), rtol=0, atol=1e-12)


@pytest.mark.parametrize("name", sorted(GRAPHS))
def test_gap_certifies_distance_along_the_run(name):
    D, lmax = GRAPHS[name]()
    x = RNG.normal(size=(D.shape[0], 3))
    zs = oo.prox_tv_exact(x, 0.3, D)
    prev = None
    for k in (1, 2, 5, 10, 30, 100, 300):
        r = oo.prox_tv_fgp(x, 0.3, D, lmax, tol=0, maxit=k)
        assert r["niter"] == k and r["crit"] == "MAXIT"
        if prev is not None:                               # a prefix of the longer run
            np.testing.assert_array_equal(r["objective"][:prev.size], prev)
        prev = r["objective"]
        assert np.all(r["gap"] >= -1e-12 * r["objective"])
        assert np.linalg.norm(r["z"] - zs) <= np.sqrt(2 * max(r["gap"][-1], 0)) + 1e-9


@pytest.mark.parametrize("name", sorted(GRAPHS))
def test_gap_identity(name):
    D, lmax = GRAPHS[name]()
    x = RNG.normal(size=(D.shape[0], 2))
    for k in (1, 7, 40):
        r = oo.prox_tv_fgp(x, 0.5, D, lmax, tol=0, maxit=k)
        z = r["z"]
        dual = 0.5 * np.sum(x * x) - 0.5 * np.sum(z * z)
        P = r["objective"][-1]
        assert abs(r["gap"][-1] - (P - dual)) <= 1e-12 * max(abs(P), 1.0)
        g = D.T @ z
        assert abs(P - (0.5 * np.sum((x - z) ** 2) + 0.5 * np.abs(g).sum())) <= 1e-13 * abs(P)


@pytest.mark.parametrize("W", [tg.geometric(), tg.disconnected()], ids=["connected", "disconnected"])
def test_large_gamma_gives_component_means(W):
    D = do.differential_operator(W)
    x = RNG.normal(size=(W.shape[0], 2))
    bound = tg.mean_bound(W, D, x)
    zs = oo.prox_tv_exact(x, 2 * bound, D)
    np.testing.assert_allclose(zs, tg.component_means(W, x), rtol=0, atol=1e-10)
    # and not below the bound
    assert np.abs(oo.prox_tv_exact(x, 0.5 * bound, D) - tg.component_means(W, x)).max() > 1e-6


def test_stop_rule_edge_cases():
    D, lmax = GRAPHS["weighted"]()
    x = np.ones(D.shape[0])
    r = oo.prox_tv_fgp(x, 0.3, D, lmax)                   # P_0 = P_1 = 0
    assert (r["niter"], r["crit"]) == (1, "RTOL")
    np.testing.assert_array_equal(r["z"][:, 0], x)
    r = oo.prox_tv_fgp(x, 0.3, D, lmax, tol=0, maxit=7)   # tol = 0 runs to maxit
    assert (r["niter"], r["crit"]) == (7, "MAXIT")
    y = RNG.normal(size=D.shape[0])
    r = oo.prox_tv_fgp(y, 0.3, D, lmax, tol=0, maxit=25)
    assert (r["niter"], r["crit"]) == (25, "MAXIT")
    r = oo.prox_tv_fgp(y, 0.3, D, lmax, tol=1e9, maxit=25)  # RTOL at the first test
    assert (r["niter"], r["crit"]) == (1, "RTOL")
    r = oo.prox_tv_fgp(y, 0.3, D, lmax, tol=1e9, maxit=1)   # maxit is checked second
    assert (r["niter"], r["crit"]) == (1, "MAXIT")


@pytest.mark.parametrize("name", sorted(GRAPHS))
def test_recorded_tolerances(name):
    """The drift the module docstring records: float64 with only the order of the sums
    changed, and float32 storage against float64, at the device tests' iteration counts."""
    D, lmax = GRAPHS[name]()
    x = np.random.default_rng(7).normal(size=(D.shape[0], 3))
    scale = np.abs(x).max()
    for k in (1, 2, 10, 50):
        ref = oo.prox_tv_fgp(x, 0.3, D, lmax, tol=0, maxit=k)
        rev = oo.prox_tv_fgp(x, 0.3, D, lmax, tol=0, maxit=k, order="reverse")
        f32 = oo.prox_tv_fgp(x, 0.3, D, lmax, tol=0, maxit=k, dtype=np.float32)
        assert np.abs(rev["z"] - ref["z"]).max() <= 1e-3 * oo.F64_Z * scale
        for key in ("objective", "gap"):
            assert np.abs(rev[key] - ref[key]).max() <= 1e-3 * oo.F64_HIST * np.abs(ref[key]).max()
        assert np.abs(f32["z"] - ref["z"]).max() <= 0.1 * oo.F32_Z * scale


def test_a_hooks_scaled_identity():
    """A = s I with nu = s^2 is the A = None iteration at gamma s."""
    D, lmax = GRAPHS["weighted"]()
    x = RNG.normal(size=(D.shape[0], 2))
    s = 1.7
    a = oo.prox_tv_fgp(x, 0.2, D, lmax, A=lambda v: s * v, At=lambda v: s * v, nu=s * s,
                       tol=0, maxit=30)
    b = oo.prox_tv_fgp(x, 0.2 * s, D, lmax, tol=0, maxit=30)
    np.testing.assert_allclose(a["z"], b["z"], rtol=0, atol=1e-12)


def test_diagonal_a_converges_to_its_prox():
    """A = At = diag(d): the gap certifies the distance to BVLS's solution of the dual with
    K* = diag(d) D."""
    D, lmax = GRAPHS["weighted"]()
    n = D.shape[0]
    d = np.random.default_rng(9).uniform(0.5, 1.5, n)
    x = RNG.normal(size=(n, 1))
    K_star = sparse.diags(d) @ D                            # K* = A* D
    zs = oo.prox_tv_exact(x, 0.3, K_star)
    r = oo.prox_tv_fgp(x, 0.3, D, lmax, A=lambda v: d[:, None] * v, At=lambda v: d[:, None] * v,
                       nu=float(d.max() ** 2), tol=0, maxit=400)
    assert np.linalg.norm(r["z"] - zs) <= np.sqrt(2 * r["gap"][-1]) + 1e-9
