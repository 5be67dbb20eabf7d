"""Float64 NumPy / SciPy-sparse restatement of classification_tikhonov_simplex
(pygsp/learning.py:42-180) in the operation order of csrc/simplex.cu: the sort-free projection
the kernel uses (Michelot), ``L y`` by linearity from ``L x_k`` and ``L x_{k-1}`` (one product
with L per iteration), the objective of x_k taken from the same ``L x_k``, and the stop rule of
pyunlocbox's ``solve`` as oracle/unlocbox_standin.py states it.  Checked against the unmodified
reference run with that stand-in by tests/test_oracle_simplex.py."""
import numpy as np
from scipy import sparse

CRITS = {1: "ATOL", 2: "DTOL", 3: "RTOL", 4: "XTOL", 5: "MAXIT"}


def proj_simplex(V):
    """Euclidean projection of every row of V onto {x >= 0, sum x = 1}: Michelot's active set,
    theta = (sum of the active values - 1) / their number, dropping values <= theta until the
    set is stable."""
    V = np.asarray(V, dtype=np.float64)
    act = np.ones(V.shape, dtype=bool)
    while True:
        theta = (np.where(act, V, 0.0).sum(axis=1) - 1.0) / np.maximum(act.sum(axis=1), 1)
        keep = act & (V > theta[:, None])
        if (keep == act).all():
            break
        act = keep
    return np.maximum(V - theta[:, None], 0.0)


def labels_of(y, M):
    """The int labels the engine passes: y[~M] = 0, truncated to int, -1 where M is False;
    and the number of classes (max label + 1, as the reference's _to_logits)."""
    M = np.asarray(M).astype(bool)
    y = np.array(y, dtype=np.float64, copy=True)
    y[~M] = 0
    lab = y.astype(int)
    C = int(lab.max()) + 1
    lab[~M] = -1
    return lab, C


def objective(L, X, lab, tau, LX=None):
    LX = L @ X if LX is None else LX
    M = lab >= 0
    Y = np.zeros_like(X)
    Y[np.flatnonzero(M), lab[M]] = 1
    fit = (X - Y)[M]
    return tau * np.sum(X * LX) + np.sum(fit * fit)


def solve(L, y, M, tau=0.1, lmax=None, atol=None, dtol=None, rtol=1e-3, xtol=None, maxit=200):
    """Returns (sol, niter, crit, objective history f_0 .. f_niter)."""
    L = sparse.csr_matrix(L)
    lab, C = labels_of(y, M)
    n = L.shape[0]
    mask = lab >= 0
    Y = np.zeros((n, C))
    Y[np.flatnonzero(mask), lab[mask]] = 1
    step = 0.5 / (1 + tau * lmax)
    x, xp = Y.copy(), Y.copy()
    lx = L @ x
    lxp = lx
    t = 1.0
    obj = []
    k = 0
    while True:
        cur = objective(L, x, lab, tau, lx)
        obj.append(cur)
        if k >= 1:
            last, crit = obj[-2], 0
            if atol is not None and cur < atol:
                crit = 1
            if dtol is not None and abs(cur - last) < dtol:
                crit = 2
            if rtol is not None:
                div = cur if cur != 0 else (last if last != 0 else 1.0)
                if abs((cur - last) / div) < rtol:
                    crit = 3
            if xtol is not None and np.linalg.norm(x - xp) / np.sqrt(x.size) < xtol:
                crit = 4
            if maxit is not None and k >= maxit:
                crit = 5
            if crit:
                return x, k, CRITS[crit], np.array(obj)
        tn = (1.0 + np.sqrt(1.0 + 4.0 * t * t)) / 2.0
        beta = (t - 1.0) / tn
        t = tn
        yk = x + beta * (x - xp)
        ly = (1.0 + beta) * lx - beta * lxp
        grad = 2.0 * (np.where(mask[:, None], yk - Y, 0.0) + tau * ly)
        x, xp = proj_simplex(yk - step * grad), x
        lx, lxp = L @ x, lx
        k += 1


def residual(L, X, lab, tau, lmax):
    """Fixed-point residual ||X - proj(X - step grad f(X))|| of a minimiser."""
    L = sparse.csr_matrix(L)
    mask = lab >= 0
    Y = np.zeros_like(X)
    Y[np.flatnonzero(mask), lab[mask]] = 1
    step = 0.5 / (1 + tau * lmax)
    grad = 2.0 * (np.where(mask[:, None], X - Y, 0.0) + tau * (L @ X))
    return np.linalg.norm(X - proj_simplex(X - step * grad))
