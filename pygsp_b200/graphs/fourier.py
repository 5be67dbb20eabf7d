"""Graph Fourier basis: partial or full eigendecomposition of the Laplacian on the device.

Mirror of ``pygsp/graphs/fourier.py`` (:1-264): ``U``, ``e``, ``coherence``,
``compute_fourier_basis``, ``gft`` and ``igft``, mixed into :class:`Graph`.  The basis lives
in HBM in the graph's dtype; ``G.U`` / ``G.e`` are host copies made once.

Two solvers, chosen from the request (no user option):

* **dense** -- the full basis, bases of more than N/4 vectors and small graphs: L is densified
  on the device and diagonalised by ``torch.linalg.eigh`` in float64 (cuSOLVER, standing in
  for the reference's LAPACK ``eigh``, fourier.py:171-172);
* **ChFSI** -- Chebyshev-filtered subspace iteration (Zhou & Saad 2007) for the smallest k
  eigenpairs of a large graph, where the reference calls ``eigsh(L, k, which='SM')``
  (fourier.py:173-175).  Its filter is the engine's fused recurrence step
  (``gsp_cheby_step_*`` with no accumulator); orthonormalisation, Rayleigh-Ritz and residuals
  are the block kernels of csrc/block.cu; only b x b matrices (b = k plus guard vectors) are
  factorised, in float64 on the host.

Column signs, and the basis inside a repeated eigenvalue, are whatever the solver returns.
The reference's sign fix (fourier.py:185, ``np.abs(U[0, 0]).sum() < 0``) never fires and is
not reproduced.
"""
import numpy as np

from .. import _native as nat

# Dense solver at or below this many vertices, ChFSI above (for k <= N / 4).  H100 SXM, 400 W
# power limit, k = 16 (tools/fourier_probe.py, DESIGN.md section 4.6): dense is faster at 1024,
# equal at 2048, 4x slower at 4096.
DENSE_CROSSOVER = 2048
# Largest Chebyshev filter degree of a ChFSI iteration: of 20 / 40 / 60 / 100, 100 was fastest
# for k = 16 and k = 64 on the 1e6-vertex config-2 graph (same card, DESIGN.md section 4.6).
FILTER_DEGREE = 100
# Largest ratio between the filter's gains at 0 and at the cut-off a, i.e. the condition
# number the filter may give the block; CholeskyQR2 in the block's dtype must absorb it.
_FILTER_RANGE = {"f32": 1e3, "f64": 1e6}
MAX_ITERATIONS = 1000
_TILED_WIDTHS = (8, 16, 32, 64, 128)


class FourierMixIn:

    def _check_fourier_properties(self, name, desc):
        if getattr(self, "_" + name) is None:
            self.logger.warning("The {} G.{} is not available, we need to "
                                "compute the Fourier basis. Explicitly call "
                                "G.compute_fourier_basis() once beforehand "
                                "to suppress the warning.".format(desc, name))
            self.compute_fourier_basis()
        return getattr(self, "_" + name)

    def _clear_fourier_basis(self):
        self._U = None
        self._U_host = None
        self._e = None
        self._coherence = None

    @property
    def U(self):
        r"""Fourier basis (eigenvectors of the Laplacian), a host ndarray (N, k)."""
        self._check_fourier_properties("U", "Fourier basis")
        if self._U_host is None:
            self._U_host = self._U.cpu().numpy()
        return self._U_host

    @property
    def e(self):
        r"""Eigenvalues of the Laplacian in ascending order (float64 host ndarray)."""
        return self._check_fourier_properties("e", "eigenvalues vector")

    @property
    def coherence(self):
        r"""Coherence of the Fourier basis, max |U|, in [1/sqrt(N), 1] (full basis only)."""
        return self._check_fourier_properties("coherence", "Fourier basis coherence")

    def compute_fourier_basis(self, n_eigenvectors=None, *, seed=0):
        r"""Compute the (partial) Fourier basis of the graph (cached; fourier.py:97-195).

        ``n_eigenvectors`` smallest eigenpairs of L (all if None).  Nothing is done if a basis
        with at least that many vectors exists.  The full basis also sets ``G.lmax`` (method
        'fourier') and ``G.coherence``.  A partial basis of a large graph is computed by
        Chebyshev-filtered subspace iteration from a start block that is a counter-based
        function of ``seed`` (reproducible); raises ``ValueError`` if it does not converge, or
        if a dense eigendecomposition does not fit in device memory.
        """
        torch = nat.require_cuda()
        n = self.n_vertices
        if n_eigenvectors is None:
            n_eigenvectors = n
        k = int(n_eigenvectors)
        if not 1 <= k <= n:
            raise ValueError("n_eigenvectors must be in [1, N = {}], got {}.".format(n, k))
        if self._U is not None and k <= len(self._e):
            return

        if n ** 2 * k > 3000 ** 3:
            self.logger.warning(
                "Computing the {0} eigendecomposition of a large matrix ({1} x"
                " {1}) is expensive. Consider decreasing n_eigenvectors "
                "or, if using the Fourier basis to filter, using a "
                "polynomial filter instead.".format("full" if k == n else "partial", n))

        if k == n or k > n / 4 or n <= DENSE_CROSSOVER:
            e, U = self._fourier_dense(k)
        else:
            e, U = self._fourier_chfsi(k, seed=seed)

        bound = self._get_upper_bound()
        slack = 1e-5 if self.dtype == torch.float64 else 1e-5 * abs(bound)
        assert -slack < e[0] < slack, e[0]
        e[0] = 0
        assert e[-1] <= bound + slack, (e[-1], bound)
        assert np.max(e) == e[-1]
        self._U, self._U_host, self._e = U, None, e
        if k == n:
            self._lmax = float(e[-1])
            self._lmax_method = "fourier"
            self._coherence = float(U.abs().max().item())

    # ------------------------------------------------------------------- transforms
    def gft(self, s):
        r"""Graph Fourier transform U^T s (fourier.py:197-230).

        Contraction over the first axis: any trailing shape.  NumPy in -> NumPy out, CUDA
        tensor in -> CUDA tensor out (graph dtype).
        """
        from ..filters import approximations as apx
        s = self._check_signal(s)
        U = self._device_basis()
        x, _, kind = apx._as_device_block(apx._GraphView(self.L), s)
        out = block_gram(U, x).to(self.dtype).reshape((U.shape[1],) + tuple(s.shape[1:]))
        return apx._leave_device(out, kind)

    def igft(self, s_hat):
        r"""Inverse graph Fourier transform U s_hat (fourier.py:232-264).

        The first dimension of ``s_hat`` is ``len(G.e)``: N for the full basis, k for a partial
        one (the reference accepts only N).
        """
        from ..filters import approximations as apx
        torch = nat.require_cuda()
        U = self._device_basis()
        if not torch.is_tensor(s_hat):
            s_hat = np.asanyarray(s_hat)
        if s_hat.shape[0] != U.shape[1]:
            self._check_signal(s_hat)          # the reference's ValueError
            raise ValueError("First dimension must be the number of Fourier modes "
                             "len(G.e) = {}, got {}.".format(U.shape[1], tuple(s_hat.shape)))
        x, _, kind = apx._as_device_block(apx._GraphView(self.L), s_hat)
        out = block_combine(U, x.double()).reshape((self.n_vertices,) + tuple(s_hat.shape[1:]))
        return apx._leave_device(out, kind)

    def _device_basis(self):
        self._check_fourier_properties("U", "Fourier basis")
        return self._U

    # ---------------------------------------------------------------------- solvers
    def _fourier_dense(self, k):
        """Smallest k eigenpairs by a dense float64 eigh on the device."""
        torch = nat.require_cuda()
        n, L = self.n_vertices, self.L
        # the dense matrix, eigh's copy of it (the eigenvectors) and its workspace (~2 N^2)
        need = 4 * n * n * 8
        free, _ = torch.cuda.mem_get_info(self.device)
        if need > free:
            raise ValueError(
                "The dense eigendecomposition of this {0} x {0} Laplacian needs about {1:.1f} GB "
                "of device memory ({2:.1f} GB free). Pass n_eigenvectors to compute a partial "
                "basis.".format(n, need / 2 ** 30, free / 2 ** 30))
        with torch.cuda.device(self.device):
            dense = L.to_dense()
            e, U = torch.linalg.eigh(dense)
            del dense
            U = U[:, :k].to(self.dtype).contiguous()
        return e[:k].cpu().numpy(), U

    def _fourier_chfsi(self, k, *, seed=0, degree=None, max_iter=None, stats=None):
        """Smallest k eigenpairs by Chebyshev-filtered subspace iteration.

        Iteration: filter the block X by a Chebyshev polynomial that amplifies [0, a] and damps
        [a, b_up] (a = largest Ritz value, b_up = _get_upper_bound(), a guaranteed bound);
        orthonormalise (CholeskyQR2); Rayleigh-Ritz; stop when the first k residuals
        ||L u_i - theta_i u_i|| are <= tol * b_up.  The degree is ``degree`` (FILTER_DEGREE)
        unless the gain ratio between 0 and a would exceed what the block's precision
        resolves; then it is lowered.  ``stats`` (a dict) receives the
        iteration and filter-step counts.
        """
        torch = nat.require_cuda()
        n = self.n_vertices
        m = FILTER_DEGREE if degree is None else int(degree)
        cap = MAX_ITERATIONS if max_iter is None else int(max_iter)
        tol = 1e-10 if self.dtype == torch.float64 else 1e-5
        b = block_width(k, n)
        upper = float(self._get_upper_bound())
        rng = _Seeds(seed)
        X = block_random(n, b, rng.next(), self.dtype, self.device)
        X = self._orthonormalize(X, rng)
        X, LX, theta = self._rayleigh_ritz(X)
        steps = 0
        for it in range(1, cap + 1):
            a = min(float(theta[-1]), 0.95 * upper)
            # gain at 0 relative to [a, upper]: T_deg((upper + a) / (upper - a)); keep it within
            # the range the block's precision resolves
            width = np.arccosh((upper + a) / (upper - a))
            deg = int(max(2, min(m, np.arccosh(_FILTER_RANGE[self._sfx]) // width)))
            X = self._chebyshev_filter(X, deg, a, upper)
            steps += deg
            X = self._orthonormalize(X, rng)
            X, LX, theta = self._rayleigh_ritz(X)
            res = np.sqrt(np.maximum(block_residual(X, LX, theta), 0))
            if stats is not None:
                stats.update(iterations=it, filter_steps=steps, block_width=b,
                             max_residual=float(res[:k].max()))
            if np.all(res[:k] <= tol * upper):
                return theta[:k].copy(), X[:, :k].contiguous()
        raise ValueError("The Chebyshev-filtered subspace iteration did not converge in {} "
                         "iterations.".format(cap))

    def _largest_eigenvector(self, *, seed=0, max_iter=None):
        """Eigenvector of the largest eigenvalue of L as a float64 host array (unit norm).

        What graph_multiresolution down-samples with (reduction.py:271-275): the last column of a
        full basis when there is one; a dense float64 ``eigh`` for small graphs; otherwise
        Chebyshev-filtered subspace iteration on the reflected operator ``b_up I - L`` (its
        smallest eigenpair is L's largest), through the same fused step with alpha and beta
        transformed, from a start block that is a counter-based function of ``seed``.  Stops when
        ``||L v - theta v|| <= tol b_up`` (tol 1e-10 in float64, 1e-5 in float32).
        """
        torch = nat.require_cuda()
        n = self.n_vertices
        if self._U is not None and len(self._e) == n:
            return self._U[:, -1].double().cpu().numpy()
        if n <= DENSE_CROSSOVER:
            with torch.cuda.device(self.device):
                _, U = torch.linalg.eigh(self.L.to_dense())
            return U[:, -1].cpu().numpy()
        cap = MAX_ITERATIONS if max_iter is None else int(max_iter)
        tol = 1e-10 if self.dtype == torch.float64 else 1e-5
        b = block_width(1, n)
        upper = float(self._get_upper_bound())
        rng = _Seeds(seed)
        X = block_random(n, b, rng.next(), self.dtype, self.device)
        X = self._orthonormalize(X, rng)
        X, LX, theta = self._rayleigh_ritz(X)
        for _ in range(cap):
            # spectrum of b_up I - L on the block: upper - theta; damp [a, upper] of it
            a = min(upper - float(theta[0]), 0.95 * upper)
            width = np.arccosh((upper + a) / (upper - a))
            deg = int(max(2, min(FILTER_DEGREE, np.arccosh(_FILTER_RANGE[self._sfx]) // width)))
            X = self._chebyshev_filter(X, deg, a, upper, reflect=True)
            X = self._orthonormalize(X, rng)
            X, LX, theta = self._rayleigh_ritz(X)
            res = np.sqrt(max(float(block_residual(X, LX, theta)[-1]), 0.0))
            if res <= tol * upper:
                return X[:, -1].double().cpu().numpy()
        raise ValueError("The Chebyshev-filtered subspace iteration for the largest eigenvector "
                         "did not converge in {} iterations.".format(cap))

    def _apply_laplacian(self, X):
        """L X by the recurrence step (alpha = 1, beta = 0): the tiled kernel where it applies."""
        torch = nat.require_cuda()
        L, n, b = self.L, self.n_vertices, X.shape[1]
        Y = torch.empty_like(X)
        zero = np.zeros(1)
        with torch.cuda.device(self.device):
            nat.call("gsp_cheby_step_" + self._sfx, nat.i32(1), nat.i64(0), nat.i64(n),
                     nat.i64(L.nnz), L.indptr, L.indices, L.data, X, X, Y, Y, nat.i64(n),
                     nat.i64(b), nat.i32(0), zero, zero, nat.f64(1.0), nat.f64(0.0),
                     nat.f64(0.0), L.tile_plan(b, 0), self._stream())
        return Y

    def _chebyshev_filter(self, X, m, a, upper, reflect=False):
        """p_m(L) X, p_m the Chebyshev polynomial of [a, upper] scaled to 1 at 0 (Zhou-Saad).
        ``reflect``: p_m(upper I - L) X, with alpha A x + beta x = -alpha L x + (alpha upper +
        beta) x for A = upper I - L."""
        torch = nat.require_cuda()
        L, n, b = self.L, self.n_vertices, X.shape[1]
        plan = L.tile_plan(b, 0)
        zero = np.zeros(1)
        c, e = (a + upper) / 2, (upper - a) / 2
        sigma = e / (0 - c)
        tau = 2 / sigma
        buf = torch.empty_like(X)
        x_cur, x_old = X, X
        with torch.cuda.device(self.device):
            for j in range(m):
                if j == 0:
                    alpha, beta, gamma, x_new = sigma / e, -sigma * c / e, 0.0, buf
                else:
                    sigma_next = 1 / (tau - sigma)
                    alpha = 2 * sigma_next / e
                    beta = -2 * sigma_next * c / e
                    gamma = -sigma * sigma_next
                    sigma = sigma_next
                    x_new = x_old            # row-local: x_new may overwrite x_old
                if reflect:
                    alpha, beta = -alpha, alpha * upper + beta
                nat.call("gsp_cheby_step_" + self._sfx, nat.i32(j == 0), nat.i64(0), nat.i64(n),
                         nat.i64(L.nnz), L.indptr, L.indices, L.data, x_cur, x_old, x_new, x_new,
                         nat.i64(n), nat.i64(b), nat.i32(0), zero, zero, nat.f64(alpha),
                         nat.f64(beta), nat.f64(gamma), plan, self._stream())
                x_old, x_cur = x_cur, x_new
        return x_cur

    def _orthonormalize(self, X, rng, attempts=4):
        """CholeskyQR2 with a float64 Gram; when the Cholesky factorisation fails, the block is
        orthonormalised through the Gram's eigendecomposition and its (numerically) dependent
        columns are replaced by fresh seeded vectors."""
        from scipy.linalg import solve_triangular
        b = X.shape[1]
        eye = np.eye(b)
        # largest condition number of X that one CholeskyQR2 pass orthonormalises in X's dtype
        floor = 1e-7 if X.dtype == nat.require_cuda().float64 else 1e-3
        for _ in range(attempts):
            G = None
            for _ in range(2):
                G = block_gram(X, X).cpu().numpy()
                try:
                    R = np.linalg.cholesky((G + G.T) / 2)
                except np.linalg.LinAlgError:
                    break
                d = np.diag(R)
                if not (np.all(np.isfinite(d)) and d.min() > floor * d.max()):
                    break
                X = block_combine(X, solve_triangular(R, eye, lower=True).T)
            else:
                return X
            w, V = _eigh((G + G.T) / 2)
            good = w > max(w[-1], 0) * 1e-12
            n_good = int(good.sum())
            keep = block_combine(X, V[:, good] / np.sqrt(w[good])) if n_good else X[:, :0]
            fresh = block_random(X.shape[0], b - n_good, rng.next(), X.dtype, X.device)
            X = nat.require_cuda().cat([keep, fresh], dim=1).contiguous()
        raise ValueError("The Chebyshev-filtered subspace iteration lost its block: "
                         "orthonormalisation failed.")

    def _rayleigh_ritz(self, X):
        """Ritz pairs of L on span(X) (X orthonormal): (X V, L X V, theta ascending)."""
        LX = self._apply_laplacian(X)
        H = block_gram(X, LX).cpu().numpy()
        theta, V = _eigh((H + H.T) / 2)
        return block_combine(X, V), block_combine(LX, V), theta


def _eigh(H):
    """Eigenpairs of a small symmetric matrix by LAPACK's divide and conquer (syevd): at
    b = 128 NumPy's default path is an order of magnitude slower on a many-core host."""
    from scipy.linalg import eigh
    return eigh(H, driver="evd")


class _Seeds:
    """Successive seeds of the start block and of replacement vectors."""

    def __init__(self, seed):
        self.seed = int(seed) * 0x100000 & 0xFFFFFFFFFFFFFFFF
        self.count = 0

    def next(self):
        self.count += 1
        return (self.seed + self.count - 1) & 0xFFFFFFFFFFFFFFFF


def block_width(k, n):
    """k plus max(4, k/4) guard vectors, rounded up to a width the tiled step serves."""
    want = k + max(4, -(-k // 4))
    for w in _TILED_WIDTHS:
        if want <= w:
            return min(w, n)
    return min(-(-want // 8) * 8, n)


# ------------------------------------------------------------------ block kernels
def _same_block(what, A, B):
    """ValueError unless A and B are blocks of one dtype, on one device, with as many rows: the
    kernels read both through A's element type and row count."""
    if A.dtype != B.dtype:
        raise ValueError("%s: dtypes differ (%s, %s)" % (what, A.dtype, B.dtype))
    if A.device != B.device:
        raise ValueError("%s: devices differ (%s, %s)" % (what, A.device, B.device))
    if A.shape[0] != B.shape[0]:
        raise ValueError("%s: row counts differ (%d, %d)" % (what, A.shape[0], B.shape[0]))


def block_gram(A, B):
    """A^T B (float64 device tensor) for (n, ka) and (n, kb) device blocks of one dtype."""
    torch = nat.require_cuda()
    _same_block("block_gram", A, B)
    A, B = A.contiguous(), B.contiguous()
    A2, B2 = A.reshape(A.shape[0], -1), B.reshape(B.shape[0], -1)
    C = torch.empty((A2.shape[1], B2.shape[1]), dtype=torch.float64, device=A.device)
    with torch.cuda.device(A.device):
        nat.call("gsp_block_gram_" + nat.suffix(A.dtype), nat.i64(A2.shape[0]), A2,
                 nat.i64(A2.shape[1]), B2, nat.i64(B2.shape[1]), C, nat.stream_ptr(A.device))
    return C


def block_combine(A, Q):
    """A Q in A's dtype for an (n, ka) device block and a (ka, kq) float64 matrix."""
    torch = nat.require_cuda()
    A = A.contiguous()
    Q = torch.as_tensor(Q, dtype=torch.float64, device=A.device).contiguous()
    Q2 = Q.reshape(Q.shape[0], -1)
    if A.dim() != 2 or Q2.shape[0] != A.shape[1]:
        raise ValueError("block_combine: Q has %d rows for a block of shape %s"
                         % (Q2.shape[0], tuple(A.shape)))
    Y = torch.empty((A.shape[0], Q2.shape[1]), dtype=A.dtype, device=A.device)
    with torch.cuda.device(A.device):
        nat.call("gsp_block_combine_" + nat.suffix(A.dtype), nat.i64(A.shape[0]), A,
                 nat.i64(A.shape[1]), Q2, nat.i64(Q2.shape[1]), Y, nat.stream_ptr(A.device))
    return Y


def block_residual(X, LX, theta):
    """||LX[:, j] - theta[j] X[:, j]||^2 for every column (host float64 array)."""
    torch = nat.require_cuda()
    _same_block("block_residual", X, LX)
    if X.dim() != 2 or LX.shape != X.shape:
        raise ValueError("block_residual: shapes %s and %s" % (tuple(X.shape), tuple(LX.shape)))
    theta = np.asarray(theta, dtype=np.float64).ravel()
    if theta.size != X.shape[1]:
        raise ValueError("block_residual: %d values of theta for %d columns"
                         % (theta.size, X.shape[1]))
    X, LX = X.contiguous(), LX.contiguous()
    th = torch.as_tensor(theta, device=X.device)
    out = torch.empty(X.shape[1], dtype=torch.float64, device=X.device)
    with torch.cuda.device(X.device):
        nat.call("gsp_block_residual_" + nat.suffix(X.dtype), nat.i64(X.shape[0]), X, LX, th,
                 nat.i64(X.shape[1]), out, nat.stream_ptr(X.device))
    return out.cpu().numpy()


def block_random(n, k, seed, dtype, device):
    """(n, k) block of uniform [-1, 1) values, a counter-based function of ``seed``."""
    torch = nat.require_cuda()
    X = torch.empty((n, k), dtype=dtype, device=device)
    if k:
        with torch.cuda.device(device):
            nat.call("gsp_block_random_" + nat.suffix(dtype), nat.i64(n), nat.i64(k),
                     nat.u64(seed), X, nat.stream_ptr(device))
    return X
