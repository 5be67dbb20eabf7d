"""CPU oracle for the graph total-variation prox (pygsp/optimization.py:24-103, prox_tv).

TEST INFRASTRUCTURE ONLY; nothing under ``pygsp_b200/`` imports it.  There are no goldens from
the reference: its ``prox_tv`` fails before computing anything (``ImportError`` without
pyunlocbox, ``NameError`` on ``verbose`` with it, and it reads ``G.Diff`` and an undefined
``D``).  So the checks are mathematical:

* ``prox_tv_fgp``: a NumPy / SciPy restatement of the iteration csrc/tv.cu runs (FISTA on the
  dual, the stop rule on the objective, the duality gap), in float64, or with the device's
  float32 storage (``dtype=np.float32``), with A / At hooks;
* ``prox_tv_exact``: z* = x - gamma D u*, u* from the box-constrained least-squares dual by
  ``scipy.optimize.lsq_linear(method='bvls')`` (Ne up to about 2000);
* ``tv1d_exact``: Condat's direct algorithm for the 1-D TV denoiser, an independent check on
  path graphs with unit weights.

Build D with ``oracle.difference_oracle.differential_operator``.

Tolerances of the device tests (``tests/test_optimization_gpu.py``), measured on this oracle by
``tests/test_oracle_optimization.py`` on the graphs and iteration counts those tests use
(maxit 1, 2, 10, 50, tol = 0), as the largest drift over them:

* float64, only the order of the sums changed (``order='reverse'``): z does not move (the sums
  feed only the stop test), the objective and the gap move by at most 9.2e-16 relative.  The
  device's fma contractions in the dual update and its vertex pass are roundings of the same
  size that do reach z: ``F64_Z = 1e-12`` of max|x| and ``F64_HIST = 1e-11`` relative leave three
  orders of magnitude or more above that.
* float32 storage of x, z, u and g (``dtype=np.float32``) against float64: z moves by at most
  8.4e-8 of max|x|.  ``F32_Z = 3e-5`` leaves a factor of several hundred for the device's float32
  vertex pass, whose summation order and fma differ from SciPy's float32 product here.
"""
import numpy as np
from scipy import optimize, sparse

CRITS = {1: "RTOL", 2: "MAXIT"}
F64_Z = 1e-12
F64_HIST = 1e-11
F32_Z = 3e-5


def _sum(a, order):
    a = np.asarray(a, dtype=np.float64).ravel()
    if order == "reverse":
        return float(np.cumsum(a[::-1])[-1]) if a.size else 0.0
    return float(np.sum(a))


def prox_tv_fgp(x, gamma, D, lmax, A=None, At=None, nu=1.0, tol=10e-4, maxit=200,
                dtype=np.float64, order="pairwise"):
    """FISTA on the dual of min_z 1/2 ||x - z||^2 + gamma ||D^T A z||_1.

    Returns ``dict(z, objective, gap, niter, crit)``: z_niter as (N, Nsig) float64, the
    histories P_0 .. P_niter and gap_0 .. gap_niter.  x: (N,) or (N, Nsig).  ``dtype`` is the
    storage type of x, z, u and g; the edge arithmetic is float64 and the vertex pass
    z = x - gamma D u runs in ``dtype``, as on the device.  ``order`` ('pairwise' or 'reverse')
    changes only the order of the objective and gap sums.
    """
    D = sparse.csc_matrix(D, dtype=np.float64)
    n, ne = D.shape
    X = np.asarray(x, dtype=np.float64).reshape(n, -1).astype(dtype)
    nsig = X.shape[1]
    Dv = D.astype(dtype).tocsr()
    Dt = sparse.csr_matrix(D.T.astype(dtype), dtype=np.float64)
    if A is None:
        A = At = (lambda v: v)
    tau = 1.0 / (gamma * 2.0 * lmax * nu)
    u = np.zeros((ne, nsig), dtype=dtype)
    up = u.copy()
    gp = np.zeros((ne, nsig), dtype=dtype)
    t = 1.0
    obj, gap = [], []
    k = 0
    while True:
        Du = (Dv @ u).astype(dtype)
        z = (X + (dtype(-gamma) * np.asarray(At(Du), dtype=dtype)).astype(dtype)).astype(dtype)
        g = Dt @ np.asarray(A(z), dtype=dtype).astype(np.float64)
        ud = u.astype(np.float64)
        cur = 0.5 * _sum((X.astype(np.float64) - z) ** 2, order) + gamma * _sum(np.abs(g), order)
        obj.append(cur)
        gap.append(gamma * _sum(np.abs(g) - ud * g, order))
        crit = None
        if k >= 1:
            prev = obj[-2]
            if abs(cur - prev) < tol * abs(cur) or (cur == 0 and prev == 0 and tol > 0):
                crit = "RTOL"
            if k >= maxit:
                crit = "MAXIT"
        if crit is not None:
            return dict(z=z.astype(np.float64), objective=np.array(obj), gap=np.array(gap),
                        niter=k, crit=crit)
        tn = (1.0 + np.sqrt(1.0 + 4.0 * t * t)) / 2.0
        b = (t - 1.0) / tn
        v = ud + b * (ud - up.astype(np.float64))
        kv = (1.0 + b) * g - b * gp.astype(np.float64)
        up, u = u, np.clip(v + tau * kv, -1.0, 1.0).astype(dtype)
        gp = g.astype(dtype)
        t = tn
        k += 1


def prox_tv_exact(x, gamma, D):
    """z* = x - gamma D u*, u* = argmin ||gamma D u - x|| over -1 <= u <= 1 (per column).

    u* need not be unique, z* is.  Dense bounded-variable least squares: Ne <= ~2000."""
    D = sparse.csc_matrix(D, dtype=np.float64)
    X = np.asarray(x, dtype=np.float64).reshape(D.shape[0], -1)
    if gamma == 0 or D.nnz == 0:
        return X.copy()
    M = gamma * D.toarray()
    Z = np.empty_like(X)
    for j in range(X.shape[1]):
        res = optimize.lsq_linear(M, X[:, j], bounds=(-1.0, 1.0), method="bvls", tol=1e-14)
        Z[:, j] = X[:, j] - M @ res.x
    return Z


def tv1d_exact(y, lam):
    """argmin_x 1/2 ||y - x||^2 + lam sum_i |x_{i+1} - x_i| by Condat's direct algorithm
    (L. Condat, "A direct algorithm for 1D total variation denoising", IEEE SPL 2013)."""
    y = np.asarray(y, dtype=np.float64)
    n = y.size
    out = np.empty(n)
    if n == 0:
        return out
    k = k0 = kminus = kplus = 0
    umin, umax = lam, -lam
    vmin, vmax = y[0] - lam, y[0] + lam
    while True:
        while k == n - 1:
            if umin < 0:
                while True:
                    out[k0] = vmin
                    k0 += 1
                    if k0 > kminus:
                        break
                k = kminus = k0
                vmin, umin = y[k], lam
                umax = vmin + umin - vmax
            elif umax > 0:
                while True:
                    out[k0] = vmax
                    k0 += 1
                    if k0 > kplus:
                        break
                k = kplus = k0
                vmax, umax = y[k], -lam
                umin = vmax + umax - vmin
            else:
                vmin += umin / (k - k0 + 1)
                out[k0:k + 1] = vmin
                return out
        umin += y[k + 1] - vmin
        if umin < -lam:
            while True:
                out[k0] = vmin
                k0 += 1
                if k0 > kminus:
                    break
            k = kplus = kminus = k0
            vmin = y[k]
            vmax = vmin + 2 * lam
            umin, umax = lam, -lam
            continue
        umax += y[k + 1] - vmax
        if umax > lam:
            while True:
                out[k0] = vmax
                k0 += 1
                if k0 > kplus:
                    break
            k = kplus = kminus = k0
            vmax = y[k]
            vmin = vmax - 2 * lam
            umin, umax = lam, -lam
            continue
        k += 1
        if umin >= lam:
            kminus = k
            vmin += (umin - lam) / (kminus - k0 + 1)
            umin = lam
        if umax <= -lam:
            kplus = k
            vmax += (umax + lam) / (kplus - k0 + 1)
            umax = -lam
