"""Float64 NumPy / SciPy-sparse restatement of pygsp/features.py (PyGSP 0.6.1), by two routes:

* the frame route (small N): the reference's own computation, the dense frame of every kernel
  (features.py:41, 58-59: ``g.compute_frame()`` filters ``np.identity(N)``, filter.py:599, with
  the order-30 ``cheby_op`` recurrence, approximations.py:58-114) and its row norms;
* the moment route (columns of larger graphs): the diagonal Chebyshev moments
  ``mu_n(i) = (T_n(Lt))_ii`` of chosen vertices from the recurrence on their identity columns,
  and ``||p(L) e_i||^2 = sum_n e_n mu_n(i)`` with e the plain Chebyshev coefficients of p^2,
  formed here by ``numpy.polynomial.chebyshev.chebmul`` -- independently of the engine's
  ``cheby_square_coeff``.

Checked against the unmodified PyGSP 0.6.1 by tests/test_oracle_features.py."""
import numpy as np
from numpy.polynomial import chebyshev as npcheb
from scipy import sparse


def cheby_coeff(kernel, lmax, m=30):
    """approximations.py:9-55 compute_cheby_coeff, N = m + 1 quadrature nodes."""
    N = m + 1
    a1 = a2 = lmax / 2.0                                               # :42-43
    num = np.cos(np.pi * (np.arange(N) + 0.5) / N)                     # :46-47
    return np.array([2.0 / N * np.dot(kernel(a1 * num + a2),
                                      np.cos(np.pi * o * (np.arange(N) + 0.5) / N))
                     for o in range(m + 1)])                           # :48-53


def cheby_op(L, lmax, c, S):
    """approximations.py:58-114 for one filter: c[0]/2 T_0 S + sum_k c[k] T_k(Lt) S."""
    L = sparse.csr_matrix(L)
    a1 = a2 = lmax / 2.0                                               # :93-96
    t_old = S                                                          # :98
    t_cur = (L.dot(S) - a2 * S) / a1                                   # :99
    r = 0.5 * c[0] * t_old + c[1] * t_cur                              # :103
    factor = 2 / a1 * (L - a2 * sparse.eye(L.shape[0]))                # :105
    for k in range(2, len(c)):                                         # :106-112
        t_new = factor.dot(t_cur) - t_old
        r += c[k] * t_new
        t_old, t_cur = t_cur, t_new
    return r


def norm_tig_frame(L, lmax, kernels, m=30):
    """compute_norm_tig by the frame (features.py:44-59): the (N Nf,) row norms, entry f N + j
    = ||p_f(L) e_j||; compute_frame's (N Nf, N) frame is filter.py:599-603."""
    N = L.shape[0]
    eye = np.identity(N)                                               # filter.py:599
    rows = [cheby_op(L, lmax, cheby_coeff(k, lmax, m), eye).T for k in kernels]
    return np.linalg.norm(np.concatenate(rows), axis=1, ord=2)         # features.py:59


def spectrogram_kernels(lmax, atom=None, M=100):
    """The shifted atoms of compute_spectrogram (features.py:80-89)."""
    if not atom:
        def atom(x):
            return np.exp(-M * (x / lmax) ** 2)                        # :82-83
    scale = np.linspace(0, lmax, M)                                    # :85
    return [(lambda x, s=s: atom(x - s)) for s in scale]               # :89


def spectrogram_frame(L, lmax, atom=None, M=100, m=30):
    """compute_spectrogram (features.py:62-94) by the frame: (N, M) squared norms."""
    return np.stack([norm_tig_frame(L, lmax, [k], m) ** 2
                     for k in spectrogram_kernels(lmax, atom, M)], axis=1)   # :88-91


def moments(L, lmax, order, cols):
    """mu (len(cols), 2 order + 1): mu[q, n] = (T_n(Lt))_{ii}, i = cols[q], from
    mu_{2k} = ||T_k e_i||^2 * 2 - 1 and mu_{2k+1} = 2 <T_{k+1} e_i, T_k e_i> - mu_1."""
    L = sparse.csr_matrix(L).astype(np.float64)
    N = L.shape[0]
    cols = np.asarray(cols)
    E = np.zeros((N, cols.size))
    E[cols, np.arange(cols.size)] = 1.0
    mu = np.zeros((cols.size, 2 * order + 1))
    t_old, t_cur = E, (2.0 / lmax) * (L @ E) - E
    mu[:, 0] = 1.0
    mu[:, 1] = np.sum(t_cur * t_old, axis=0)
    mu1 = mu[:, 1]
    for k in range(1, order + 1):
        mu[:, 2 * k] = 2.0 * np.sum(t_cur * t_cur, axis=0) - 1.0
        if k == order:
            break
        t_new = (4.0 / lmax) * (L @ t_cur) - 2.0 * t_cur - t_old
        mu[:, 2 * k + 1] = 2.0 * np.sum(t_new * t_cur, axis=0) - mu1
        t_old, t_cur = t_cur, t_new
    return mu


def square_norms_moments(L, lmax, kernels, cols, m=30):
    """(len(cols), len(kernels)): ||p(L) e_i||^2 for i in cols by the moment route."""
    mu = moments(L, lmax, m, cols)
    out = np.empty((len(cols), len(kernels)))
    for f, k in enumerate(kernels):
        a = cheby_coeff(k, lmax, m)
        a[0] *= 0.5                                                    # plain T_0 coefficient
        out[:, f] = mu @ npcheb.chebmul(a, a)
    return out


def avg_adj_deg(W):
    """features.py:23 with G.A = W > 0 (graph.py:726): boolean product, (N, 1)."""
    A = sparse.csr_matrix(W) > 0
    return np.asarray(np.sum(A @ A, axis=1) / (np.sum(A, axis=1) + 1.0))
