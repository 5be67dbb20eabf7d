"""The simplex-classification oracle (oracle/learning_oracle.py) against tests/golden/simplex.npz,
the output of the unmodified PyGSP 0.6.1 run with oracle/unlocbox_standin.py in place of
pyunlocbox -- no GPU needed."""
import os
import sys

import numpy as np
import pytest

from conftest import csr_from, load_golden
from oracle import learning_oracle as lo

CASES = [str(c) for c in load_golden("simplex")["cases"]]
REF = os.environ.get("PYGSP_REFERENCE")


def relmax(a, b):
    return np.abs(np.asarray(a) - b).max() / max(np.abs(b).max(), 1e-300)


def problem(z, c):
    return csr_from(z, c + "_L"), z[c + "_y"], z[c + "_M"], float(z[c + "_tau"]), float(z[c + "_lmax"])


@pytest.mark.parametrize("c", CASES)
def test_oracle_reproduces_the_reference(golden, c):
    z = golden("simplex")
    L, y, M, tau, lmax = problem(z, c)
    sol, niter, crit, obj = lo.solve(L, y, M, tau, lmax)
    assert niter == int(z[c + "_niter"]) and crit == str(z[c + "_crit"])
    assert sol.shape == z[c + "_sol"].shape
    assert relmax(sol, z[c + "_sol"]) <= 1e-12
    assert relmax(obj, z[c + "_obj"]) <= 1e-12
    for k in (1, 2, 17):
        sk, nk, ck, _ = lo.solve(L, y, M, tau, lmax, rtol=None, maxit=k)
        assert nk == k and ck == "MAXIT"
        assert relmax(sk, z["%s_sol%d" % (c, k)]) <= 1e-12


@pytest.mark.parametrize("c", CASES)
def test_converged_fixture_is_a_fixed_point(golden, c):
    z = golden("simplex")
    L, y, M, tau, lmax = problem(z, c)
    X = z[c + "_conv"]
    lab, C = lo.labels_of(y, M)
    assert X.shape == (L.shape[0], C)
    assert lo.residual(L, X, lab, tau, lmax) <= 1e-10 * np.linalg.norm(X)
    assert np.all(X >= 0) and np.allclose(X.sum(axis=1), 1, atol=1e-14)


def adversarial_rows():
    rng = np.random.default_rng(0)
    rows = [np.array([[0.3, 0.3, 0.3, 0.3]]),                   # equal values
            np.array([[0.5, 0.5, -1.0, 2.0, 2.0]]),             # ties at the top
            np.array([[0.2, 0.3, 0.5], [1.0, 0.0, 0.0]]),       # already on the simplex
            np.array([[7.0], [-3.0], [0.0]]),                   # C = 1
            np.array([[1e8, 1.0, -1e8, 1e8 - 1]]),              # 1e+8 magnitudes
            np.array([[1e-8, 2e-8, -1e-8, 0.0]]),               # 1e-8 magnitudes
            np.array([[5.0, 0.1, 0.2, 0.1]]),                   # one dominant entry
            rng.standard_normal((20, 200)),                     # C = 200
            np.round(rng.standard_normal((50, 7)), 1)]          # many ties
    return rows


def sort_projection(V):
    """The textbook sort-based projection (an independent restatement)."""
    U = -np.sort(-V, axis=1)
    css = np.cumsum(U, axis=1) - 1
    k = np.arange(1, V.shape[1] + 1)
    rho = (U - css / k > 0).sum(axis=1)
    theta = css[np.arange(V.shape[0]), rho - 1] / rho
    return np.maximum(V - theta[:, None], 0)


@pytest.mark.parametrize("i", range(len(adversarial_rows())))
def test_projection_equals_a_sort_based_projection(i):
    V = adversarial_rows()[i]
    P = lo.proj_simplex(V)
    scale = max(1.0, np.abs(V).max())
    assert np.abs(P - sort_projection(V)).max() <= 1e-15 * scale * V.shape[1]
    assert np.all(P >= 0)
    assert np.abs(P.sum(axis=1) - 1).max() <= 1e-15 * scale * V.shape[1]


@pytest.fixture(scope="module")
def reference():
    """The reference's learning module with the stand-in installed (sys.modules restored after)."""
    if not REF:
        pytest.skip("PYGSP_REFERENCE is not set")
    saved_path, saved_mods = list(sys.path), dict(sys.modules)
    sys.path.insert(0, REF)
    from oracle import unlocbox_standin
    unlocbox_standin.install()
    from pygsp import learning
    yield learning
    sys.path[:] = saved_path
    for name in list(sys.modules):
        if name not in saved_mods:
            del sys.modules[name]


def reference_proj_simplex(learning):
    """The reference's own nested proj_simplex, taken from the functions it hands to solve."""
    import pyunlocbox
    captured = {}
    real = pyunlocbox.solvers.solve

    def capture(functions, x0, solver, **kwargs):
        captured["prox"] = functions[1]._prox
        return {"sol": x0}

    class G:
        lmax = 2.0
        L = np.eye(2)
    pyunlocbox.solvers.solve = capture
    try:
        learning.classification_tikhonov_simplex(G, np.array([0.0, 1.0]), np.array([True, True]))
    finally:
        pyunlocbox.solvers.solve = real
    return lambda V: captured["prox"](V, 1.0)


def test_projection_equals_the_references(reference):
    proj = reference_proj_simplex(reference)
    for V in adversarial_rows():
        scale = max(1.0, np.abs(V).max())
        assert np.abs(lo.proj_simplex(V) - proj(V)).max() <= 1e-15 * scale * V.shape[1]


@pytest.mark.parametrize("c", CASES)
def test_standin_reproduces_the_fixtures(reference, golden, c):
    from scipy import sparse
    z = golden("simplex")
    L, y, M, tau, lmax = problem(z, c)

    class G:
        pass
    G.L, G.lmax = sparse.csr_matrix(L), lmax
    sol = reference.classification_tikhonov_simplex(G, y, M, tau=tau, verbosity="NONE")
    np.testing.assert_array_equal(sol, z[c + "_sol"])
    sol17 = reference.classification_tikhonov_simplex(G, y, M, tau=tau, rtol=None, maxit=17)
    np.testing.assert_array_equal(sol17, z[c + "_sol17"])
