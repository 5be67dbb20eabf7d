"""CPU oracle for the Chebyshev filtering hot path of PyGSP 0.6.1.

TEST INFRASTRUCTURE ONLY.  Nothing under ``pygsp_b200/`` imports this module;
only ``tests/``, ``__graft_entry__.smoke()`` and the ``cpu_baseline`` /
``--impl reference`` legs of ``bench.py`` may.  It is the *checker*, never the
thing measured as the product or shipped.

Parity status: PINNED.  ``tests/test_oracle_golden.py`` checks every function
below against fixtures under ``tests/golden/`` that were produced by importing
the real reference (PyGSP 0.6.1 @ 4716b12) with
``tests/golden/make_golden.py`` -- the Logo README example, the
``Sensor(123, seed=42)`` fixtures of the reference's own test-suite, the
Laplacian / lmax known-answer matrices of ``pygsp/tests/test_graphs.py`` and
the doctest golden ``0.27649`` of ``pygsp/filters/filter.py:255``.

The arithmetic of the reference path physically executes inside SciPy
(``scipy.sparse._sparsetools.csr_matvecs`` -- an un-vendored dependency,
``pyproject.toml:47-50`` lists it un-pinned; this image has scipy 1.18.1).
Its published algorithm is the textbook row-wise CSR product
``Y[i,:] += A[i,j] * X[j,:]`` in stored order; :func:`csr_spmm` restates it
in NumPy and ``oracle/cheby_oracle.c`` restates it in plain C.  By default the
recurrence below multiplies with ``scipy.sparse`` itself (the very engine the
reference calls), and the tests cross-check the three against each other.

Everything here is float64, exactly like the reference (``np.zeros`` default
dtype, ``approximations.py:89-91``).
"""

import numpy as np
from scipy import sparse


# ---------------------------------------------------------------------------
# graph side  (reference: pygsp/graphs/graph.py)
# ---------------------------------------------------------------------------

def canonical_adjacency(adjacency):
    """Adjacency -> CSR without stored zeros.

    Follows ``Graph.__init__`` (graph.py:98-128): anything is turned into a
    ``csr_matrix`` (duplicates summed, indices sorted by scipy's converters),
    must be square, must not hold NaN/Inf, stored zeros are removed.
    """
    if not sparse.issparse(adjacency):
        adjacency = np.asanyarray(adjacency)
    if adjacency.ndim != 2 or adjacency.shape[0] != adjacency.shape[1]:
        raise ValueError("Adjacency: must be a square matrix.")
    W = sparse.csr_matrix(adjacency, copy=True)
    total = W.sum()
    if np.isnan(total):
        raise ValueError("Adjacency: there is a Not a Number (NaN).")
    if np.isinf(total):
        raise ValueError("Adjacency: there is an infinite value.")
    W.sum_duplicates()
    W.eliminate_zeros()
    W.sort_indices()
    return W


def is_directed(W):
    """graph.py:368-405 -- directed iff W differs from its transpose."""
    return (W != W.T).nnz != 0


def count_edges(W, directed):
    """graph.py:133-140 -- undirected edges are counted once, loops once."""
    if directed:
        return int(W.nnz)
    loops = int(np.count_nonzero(W.diagonal()))
    return (W.nnz - loops) // 2 + loops


def weighted_degree(W, directed):
    """graph.py:830-838 -- column sums (undirected) or (in+out)/2 (directed)."""
    col = np.asarray(W.sum(axis=0)).ravel()
    if not directed:
        return col
    row = np.asarray(W.sum(axis=1)).ravel()
    return (col + row) / 2


def degree(W, directed):
    """graph.py:772-781 -- number of neighbours; (in+out)/2 when directed."""
    if not directed:
        return W.getnnz(axis=1)
    return (W.getnnz(axis=0) + W.getnnz(axis=1)) / 2


def symmetrize_average(W):
    """utils.py:247-248 -- (W + W^T)/2; sums that cancel exactly vanish."""
    S = ((W + W.T) / 2).tocsr()
    S.eliminate_zeros()
    S.sort_indices()
    return S


def laplacian(W, lap_type="combinatorial"):
    """Graph Laplacian as canonical CSR (graph.py:510-630).

    Built WITHOUT scipy's sparse binops so that it is an independent check of
    them: every row of L is the sorted merge of the negated (and, for the
    normalized Laplacian, degree-scaled) off-diagonal entries of the
    symmetrised adjacency with one diagonal entry; entries that evaluate to
    exactly 0.0 are not stored (scipy's binops / ``eliminate_zeros`` drop
    them, graph.py:619-628), so an isolated vertex owns an empty row.
    """
    W = W.tocsr()
    directed = is_directed(W)
    dw = weighted_degree(W, directed)
    Ws = symmetrize_average(W) if directed else W
    n = W.shape[0]
    rows = np.repeat(np.arange(n), np.diff(Ws.indptr))
    cols = Ws.indices
    vals = Ws.data.astype(np.float64)
    off = rows != cols
    loop = np.zeros(n)
    np.add.at(loop, rows[~off], vals[~off])        # w_ii (0 when no loop)

    if lap_type == "combinatorial":
        diag = dw - loop                           # graph.py:618-620
        off_vals = -vals[off]
    elif lap_type == "normalized":                 # graph.py:621-628
        d = np.zeros(n)
        connected = dw != 0
        with np.errstate(invalid="ignore"):
            d[connected] = np.power(dw[connected], -0.5)
        # (D*W)*D is evaluated left to right by scipy: (d_i * w_ij) * d_j
        off_vals = -((d[rows[off]] * vals[off]) * d[cols[off]])
        has_loop = np.zeros(n, dtype=bool)
        has_loop[rows[~off]] = True
        with np.errstate(invalid="ignore"):
            # no stored loop -> D*W*D has no diagonal entry -> I - 0 = 1 exactly
            diag = np.where(has_loop, 1.0 - (d * loop) * d, 1.0)
        diag[~connected] = 0.0
    else:
        raise ValueError("Unknown Laplacian type {}".format(lap_type))

    r = np.concatenate([rows[off], np.arange(n)])
    c = np.concatenate([cols[off], np.arange(n)])
    v = np.concatenate([off_vals, diag])
    keep = v != 0
    L = sparse.coo_matrix((v[keep], (r[keep], c[keep])), shape=(n, n)).tocsr()
    L.sort_indices()
    return L


def upper_bound(W, lap_type="combinatorial"):
    """Algebraic bound on the spectrum (graph.py:933-960).

    The fourth (Merris) bound divides by ``dw``; with an isolated vertex it is
    NaN and Python's ``min`` silently skips a trailing NaN, so the reference
    then returns the minimum of the first three.  Reproduced here.
    """
    if lap_type == "normalized":
        return 2
    if lap_type != "combinatorial":
        raise ValueError("Unknown Laplacian type {}".format(lap_type))
    directed = is_directed(W)
    dw = weighted_degree(W, directed)
    n = W.shape[0]
    bounds = [n * W.max(), 2 * dw.max()]
    if W.nnz > 0:
        coo = W.tocoo()
        bounds.append(np.max(dw[coo.row] + dw[coo.col]))
    Ws = symmetrize_average(W) if directed else W
    with np.errstate(divide="ignore", invalid="ignore"):
        merris = np.max(dw + Ws.dot(dw) / dw)
    if not np.isnan(merris):
        bounds.append(merris)
    return float(min(bounds))


def lambda_max_exact(L):
    """Largest eigenvalue of L to ~1e-10 -- the truth the estimate brackets."""
    n = L.shape[0]
    if n <= 1500:
        return float(np.linalg.eigvalsh(L.toarray())[-1])
    from scipy.sparse.linalg import eigsh
    v0 = np.random.default_rng(0).standard_normal(n)
    return float(eigsh(L.asfptype(), k=1, which="LA", tol=1e-10, v0=v0,
                       return_eigenvectors=False)[0])


def lmax_lanczos_band(L):
    """Acceptance band for ``estimate_lmax('lanczos')`` (graph.py:911-921).

    The reference runs ARPACK with tol=5e-3 from an UNSEEDED start vector and
    multiplies the Ritz value by 1.01, so its own output is not reproducible
    run to run (Logo: 13.92092 / 13.92108 / 13.92090).  What is stable is the
    bracket  lam_true <= lmax <= 1.01 * lam_true  (Ritz values never exceed the
    true eigenvalue); the lower edge is relaxed by the Ritz error tol^2.
    """
    lam = lambda_max_exact(L)
    return lam * 1.01 * (1 - 5e-3), lam * 1.01 * (1 + 1e-9)


# ---------------------------------------------------------------------------
# filter side  (reference: pygsp/filters/)
# ---------------------------------------------------------------------------

def heat_kernels(lmax, scale=10):
    """filters/heat.py:102-119 (normalize=False): min(exp(-s*x/lmax), 1)."""
    try:
        scales = list(scale)
    except TypeError:
        scales = [scale]
    return [lambda x, s=s: np.minimum(np.exp(-s * np.asarray(x) / lmax), 1)
            for s in scales]


def log_scales(lmin, lmax, n, t1=1, t2=2):
    """utils.py:312-339 -- log-spaced wavelet scales, largest first."""
    return np.exp(np.linspace(np.log(t2 / lmin), np.log(t1 / lmax), n))


def mexican_hat_kernels(lmax, Nf=6, lpfactor=20, scales=None, normalize=False):
    """filters/mexicanhat.py:55-84: one low-pass + (Nf-1) band-pass x*exp(-x)."""
    lmin = lmax / lpfactor
    if scales is None:
        scales = log_scales(lmin, lmax, Nf - 1)
    if len(scales) != Nf - 1:
        raise ValueError("len(scales) should be Nf-1.")
    kernels = [lambda x: 1.2 * np.exp(-1) * np.exp(-(np.asarray(x) / 0.4 / lmin) ** 4)]
    for t in scales:
        amp = np.sqrt(t) if normalize else 1
        kernels.append(lambda x, t=t, amp=amp: amp * (t * np.asarray(x)) * np.exp(-t * np.asarray(x)))
    return kernels


def cheby_coeff(kernels, lmax, order=30, quad=None):
    """Chebyshev-Gauss quadrature of every kernel on [0, lmax].

    approximations.py:9-55 -- c[o] = 2/Q * sum_j g(a cos(th_j) + a) cos(o th_j),
    th_j = pi (j + 1/2) / Q, a = lmax/2, Q = order+1 nodes by default.
    Returns an (Nscales, order+1) float64 array.
    """
    Q = quad if quad else order + 1
    half = lmax / 2.0
    theta = np.pi * (np.arange(Q) + 0.5) / Q
    nodes = half * np.cos(theta) + half
    out = np.empty((len(kernels), order + 1))
    for i, g in enumerate(kernels):
        gv = g(nodes)
        for o in range(order + 1):
            out[i, o] = 2.0 / Q * np.dot(gv, np.cos(o * theta))
    return out


def csr_spmm(indptr, indices, data, X):
    """Y = A X, A in CSR -- restatement of scipy's ``csr_matvecs`` in NumPy.

    For every row the products ``a_ij * X[j, :]`` are accumulated in stored
    order; ``np.add.reduceat`` over the row segments does the same sums.
    """
    X2 = X.reshape(X.shape[0], -1)
    n = len(indptr) - 1
    Y = np.zeros((n, X2.shape[1]))
    if len(indices):
        prod = data[:, None] * X2[indices]
        nonempty = np.flatnonzero(np.diff(indptr) > 0)
        Y[nonempty] = np.add.reduceat(prod, indptr[nonempty], axis=0)
    return Y.reshape((n,) + X.shape[1:])


def cheby_op(L, lmax, c, signal, spmm="scipy"):
    """Chebyshev polynomial of L applied to a signal block (approximations.py:58-114).

    r_i = 1/2 c_i0 T_0 + sum_{k>=1} c_ik T_k with T_0 = x,
    T_1 = (L x - a x)/a, T_k = (2/a)(L - a I) T_{k-1} - T_{k-2}, a = lmax/2.
    Output: (Nscales*N, Nsig) -- or (Nscales*N,) for a 1-D signal --
    filter-major row blocks.
    """
    c = np.atleast_2d(np.asarray(c, dtype=np.float64))
    nscales, M = c.shape
    if M < 2:
        raise TypeError("The coefficients have an invalid shape")
    L = L.tocsr()
    n = L.shape[0]
    x = np.asarray(signal, dtype=np.float64)
    a = float(lmax) / 2.0

    if spmm == "scipy":
        mul = L.dot
    else:
        mul = lambda v: csr_spmm(L.indptr, L.indices, L.data, v)

    t_old = x
    t_cur = (mul(x) - a * x) / a
    r = np.zeros((nscales * n,) + x.shape[1:])
    for i in range(nscales):
        r[i * n:(i + 1) * n] = 0.5 * c[i, 0] * t_old + c[i, 1] * t_cur
    for k in range(2, M):
        # (2/a)(L - aI) t = (2/a) L t - 2 t
        t_new = (2.0 / a) * mul(t_cur) - 2.0 * t_cur - t_old
        for i in range(nscales):
            r[i * n:(i + 1) * n] += c[i, k] * t_new
        t_old, t_cur = t_cur, t_new
    return r


def cheby_rect(L, lmax, bounds, signal, order=30):
    """Ideal band-pass by closed-form Chebyshev coefficients (approximations.py:117-163)."""
    bounds = np.asarray(bounds, dtype=np.float64)
    if bounds.shape != (2,):
        raise ValueError("Bounds of wrong shape.")
    x = np.asarray(signal, dtype=np.float64)
    b1, b2 = np.arccos(2.0 * bounds / lmax - 1.0)
    L = L.tocsr()
    step = lambda v: (4.0 / lmax) * L.dot(v) - 2.0 * v
    t_old = x
    t_cur = step(x) / 2.0
    r = (b1 - b2) / np.pi * x + 2.0 / np.pi * (np.sin(b1) - np.sin(b2)) * t_cur
    for k in range(2, order + 1):
        t_new = step(t_cur) - t_old
        r = r + 2.0 / (k * np.pi) * (np.sin(k * b1) - np.sin(k * b2)) * t_new
        t_old, t_cur = t_cur, t_new
    return r


def filter_signal(L, lmax, kernels, s, order=30):
    """``Filter.filter(s, method='chebyshev', order)`` (filters/filter.py:146-328).

    Shape rules: the signal is read as (N, Nsig, Nfeat); a trailing dimension
    that is neither 1 nor Nf is a *signal* dimension; Nfeat == 1 -> analysis
    (one cheby_op with all filters), Nfeat == Nf -> synthesis (sum over
    filters of single-filter cheby_ops); the result is squeezed.
    """
    n = L.shape[0]
    nf = len(kernels)
    s = np.asanyarray(s)
    if s.shape[0] != n:
        raise ValueError("First dimension must be the number of vertices "
                         "G.N = {}, got {}.".format(n, s.shape))
    if s.ndim == 1 or s.shape[-1] not in (1, nf):
        if s.ndim == 3:
            raise ValueError("Third dimension (#features) should be either 1 or the "
                             "number of filters Nf = {}, got {}.".format(nf, s.shape))
        s = s[..., None]
    feat_in = s.shape[-1]
    if s.ndim < 3:
        s = s[:, None, :]
    if s.ndim > 3:
        raise ValueError("At most 3 dimensions: #nodes x #signals x #features.")
    nsig = s.shape[1]
    c = cheby_coeff(kernels, lmax, order)

    if feat_in == 1:                                       # analysis
        r = cheby_op(L, lmax, c, s[:, :, 0])               # (nf*n, nsig)
        out = r.reshape(nf, n, nsig).transpose(1, 2, 0)    # (n, nsig, nf)
    else:                                                  # synthesis
        out = np.zeros((n, nsig))
        for i in range(nf):
            out += cheby_op(L, lmax, c[i], s[:, :, i])
        out = out[:, :, None]
    return out.squeeze()


# --------------------------------------------------------------------------- callers
# SURVEY.md 8f rank 3: reduction.interpolate / pyramid_analysis / pyramid_synthesis (direct
# branch) and learning.regression_tikhonov.  Restated on top of the oracle's own filter.
def kron_reduction(L, ind):
    """Schur complement of L onto the vertices ``ind`` (reduction.py:352-366, matrix branch)."""
    from scipy.sparse import linalg
    L = sparse.csr_matrix(L)
    n = L.shape[0]
    ind = np.asarray(ind)
    comp = np.setdiff1d(np.arange(n, dtype=int), ind)
    L_red = L[np.ix_(ind, ind)]
    L_in_out = L[np.ix_(ind, comp)]
    L_out_in = L[np.ix_(comp, ind)].tocsc()
    L_comp = L[np.ix_(comp, comp)].tocsc()
    Lnew = L_red - L_in_out.dot(linalg.spsolve(L_comp, L_out_in))
    if np.abs(Lnew - Lnew.T).sum() < np.spacing(1) * np.abs(Lnew).sum():
        Lnew = (Lnew + Lnew.T) / 2.0
    return sparse.csr_matrix(Lnew)


def _legacy_analysis(L, lmax, kernel, s, order):
    """reduction.py:26-31 ``_analysis`` for a one-filter bank and an (N, Nv) signal block;
    column j of the result is the filtered column j (the reference's reshape keeps that
    layout only for Nv == 1 -- see tests/golden/make_golden_r2.py)."""
    s = np.asarray(s, dtype=np.float64)
    cols = s.reshape(s.shape[0], -1)
    out = filter_signal(L, lmax, [kernel], cols, order=order)
    return np.asarray(out).reshape(cols.shape)


def interpolate(L, lmax, f_subsampled, keep_inds, order=100, reg_eps=0.005, K_reg=None):
    """reduction.py:150-193: alpha = K_reg f; zero-fill; Green kernel 1/(eps + x) filter."""
    n = L.shape[0]
    if K_reg is None:
        K_reg = kron_reduction(L + reg_eps * sparse.eye(n), keep_inds)
    f_subsampled = np.asarray(f_subsampled, dtype=np.float64)
    sub = f_subsampled.reshape(f_subsampled.shape[0], -1)
    full = np.zeros((n, sub.shape[1]))
    full[np.asarray(keep_inds)] = K_reg.dot(sub)
    return _legacy_analysis(L, lmax, lambda x: 1.0 / (reg_eps + x), full, order)


def pyramid_analysis(Ls, lmaxs, idxs, f, h, order=30, reg_eps=0.005, K_regs=None):
    """reduction.py:384-449.  Ls / lmaxs: Laplacian and lmax per level (levels + 1 of them),
    idxs[i] = vertices of level i kept at level i + 1, h: one kernel for all levels."""
    levels = len(Ls) - 1
    f = np.asarray(f, dtype=np.float64)
    ca, pe = [f.reshape(f.shape[0], -1)], []
    for i in range(levels):
        s_low = _legacy_analysis(Ls[i], lmaxs[i], h, ca[i], order)
        ca.append(s_low[idxs[i]])
        s_pred = interpolate(Ls[i], lmaxs[i], ca[i + 1], idxs[i], order=order, reg_eps=reg_eps,
                             K_reg=None if K_regs is None else K_regs[i])
        pe.append(ca[i] - s_pred)
    return ca, pe


def pyramid_synthesis(Ls, lmaxs, idxs, cap, pe, order=30, reg_eps=0.005, K_regs=None):
    """reduction.py:504-514, direct (not least-squares) branch."""
    levels = len(Ls) - 1
    ca = [np.asarray(cap, dtype=np.float64)]
    for i in range(levels):
        lv = levels - i - 1
        s_pred = interpolate(Ls[lv], lmaxs[lv], ca[i], idxs[lv], order=order, reg_eps=reg_eps,
                             K_reg=None if K_regs is None else K_regs[lv])
        ca.append(s_pred + pe[lv])
    return ca[levels], ca


def regression_tikhonov(L, y, M, tau=0):
    """learning.py:255-365 solved EXACTLY (sparse direct): argmin |Mx - y|^2 + tau x'Lx for
    tau > 0 (the reference runs scipy CG to rtol 1e-5 on the same system), and the harmonic
    extension L_uu x_u = -L_ul y_l for tau = 0 (:350-365)."""
    from scipy.sparse import linalg
    L = sparse.csr_matrix(L, dtype=np.float64)
    M = np.asarray(M, dtype=bool)
    y = np.array(y, dtype=np.float64)
    if tau > 0:
        y[~M] = 0
        A = (sparse.diags(M.astype(np.float64)) + tau * L).tocsc()
        return linalg.spsolve(A, y) if y.ndim == 1 else linalg.splu(A).solve(y)
    if M.size != L.shape[0]:
        raise ValueError("M should be of size [G.n_vertices,]")
    Luu = L[~M, :][:, ~M].tocsc()
    Wul = -L[~M, :][:, M]
    sol = y.copy()
    rhs = Wul.dot(y[M])
    sol[~M] = linalg.spsolve(Luu, rhs) if rhs.ndim == 1 else linalg.splu(Luu).solve(rhs)
    return sol
