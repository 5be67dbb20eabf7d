"""Float64 NumPy / SciPy-sparse restatement of Lanczos filtering (pygsp/filters/
approximations.py:228-341) with this engine's rules: one independent process per signal column,
the reference's step order, and the relative breakdown test of csrc/krylov.cu (a column stops
growing when beta_{k+1} <= 16 eps max(largest |alpha|, |beta| so far, ||A||_inf)).  Checked
against the unmodified PyGSP 0.6.1 by tests/test_oracle_lanczos.py."""
import numpy as np
from scipy import sparse

BREAKDOWN = 16.0


def norm_bound(A):
    """||A||_inf, the largest absolute row sum."""
    A = sparse.csr_matrix(A)
    return float(np.max(np.asarray(abs(A).sum(axis=1)).ravel(), initial=0.0))


def krylov(A, x, order, dtype=np.float64):
    """One Lanczos process per column of x (N, M): returns V (order, N, M), alpha, beta
    (order, M) and m (M,).  beta[k] couples vectors k - 1 and k (beta[0] = ||x_j||); entries
    past a column's breakdown are zero.  ``dtype=np.float32`` runs the whole process in
    float32 NumPy arithmetic (a bound for the engine's float32 path, whose sums are float64)."""
    eps = np.finfo(dtype).eps
    A = sparse.csr_matrix(A).astype(dtype)
    x = np.asarray(x).astype(dtype).reshape(A.shape[0], -1)
    n, M = x.shape
    anorm = norm_bound(A)
    V = np.zeros((order, n, M), dtype=dtype)
    alpha, beta = np.zeros((order, M)), np.zeros((order, M))
    m = np.zeros(M, dtype=np.int64)
    for j in range(M):
        nrm = np.linalg.norm(x[:, j])
        beta[0, j] = nrm
        if nrm == 0:
            continue
        V[0, :, j] = x[:, j] / nrm
        m[j], scale = 1, 0.0
        for k in range(order):
            q = V[k, :, j]
            r = A @ q
            if k > 0:
                r -= beta[k, j] * V[k - 1, :, j]
            alpha[k, j] = q @ r
            if k == order - 1:
                break
            r -= alpha[k, j] * q
            if k > 0:                                    # approximations.py:335
                B = V[:k + 1, :, j]
                r -= B.T @ (B @ r)
            b = np.linalg.norm(r)
            scale = max(scale, abs(alpha[k, j]))
            if b <= BREAKDOWN * eps * max(scale, anorm):
                break
            scale = max(scale, b)
            beta[k + 1, j] = b
            V[k + 1, :, j] = r / b
            m[j] = k + 2
    return V, alpha, beta, m


def tridiagonal(alpha, beta, j):
    """T_j (order x order) of column j."""
    T = np.diag(alpha[:, j])
    off = beta[1:, j]
    return T + np.diag(off, 1) + np.diag(off, -1)


def orth(V, M, order, m):
    """The reference's ||V^T V - M||_F after each step (approximations.py:314, 337), formed
    directly: the basis as it stands after step k holds vector i of signal j when
    i <= min(k, m_j - 1) and zeros elsewhere."""
    out = np.zeros(order)
    for k in range(order):
        Vk = np.zeros_like(V)
        for j in range(M):
            c = j * order + np.arange(min(k + 1, int(m[j])))
            Vk[:, c] = V[:, c]
        out[k] = np.linalg.norm(Vk.T @ Vk - M)
    return out


def lanczos(A, order, x):
    """(V, H, orth) in the reference's layout: V (N, M*order) with signal j's vector k in column
    j*order + k, H (order, M*order) with T_j in columns j*order .. j*order + order - 1."""
    x = np.asarray(x, dtype=np.float64)
    M = 1 if x.ndim == 1 else x.shape[1]
    Vb, alpha, beta, m = krylov(A, x, order)
    V = np.transpose(Vb, (1, 2, 0)).reshape(Vb.shape[1], M * order)
    H = np.zeros((order, M * order))
    for j in range(M):
        H[:, j * order:(j + 1) * order] = tridiagonal(alpha, beta, j)
    return V, H, orth(V, M, order, m)


def lanczos_op(evaluate, A, s, order=30, dtype=np.float64):
    """(Nf*N,) or (Nf*N, Nv): column j is V_j Q_j f(max(Theta_j, 0)) Q_j^T (V_j^T s_j) over the
    leading m_j x m_j block; ``evaluate`` maps Ritz values to an (Nf, m) response."""
    s = np.asarray(s, dtype=np.float64)
    one_d = s.ndim == 1
    x = s.reshape(s.shape[0], -1)
    n, nv = x.shape
    Vb, alpha, beta, m = krylov(A, x, order, dtype)
    Vb, alpha, beta = Vb.astype(np.float64), alpha.astype(np.float64), beta.astype(np.float64)
    out = None
    for j in range(nv):
        mj = int(m[j])
        if mj == 0:
            continue
        e, Q = np.linalg.eigh(tridiagonal(alpha, beta, j)[:mj, :mj])
        e[e < 0] = 0
        fe = np.atleast_2d(evaluate(e))
        if out is None:
            out = np.zeros((fe.shape[0], n, nv))
        B = Vb[:mj, :, j].T                              # (N, m_j)
        proj = Q.T @ (B.T @ x[:, j])
        for f in range(fe.shape[0]):
            out[f, :, j] = B @ (Q @ (fe[f] * proj))
    if out is None:
        out = np.zeros((np.atleast_2d(evaluate(np.zeros(1))).shape[0], n, nv))
    out = out.reshape(-1, nv)
    return out.reshape(-1) if one_d else out
