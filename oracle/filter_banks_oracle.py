"""CPU oracle for the Gabor and Modulation filter banks of PyGSP 0.6.1 (filters/gabor.py,
filters/modulation.py), restated in NumPy float64 from a given Fourier basis (e, U).

TEST INFRASTRUCTURE ONLY.  Nothing under ``pygsp_b200/`` imports this module.

Both banks have one filter per vertex.  The Modulation outputs depend on the signs of the
eigenvectors, so the tests evaluate these restatements with the engine's own basis; against the
reference's fixture they compare only sign-invariant quantities (tests/test_filter_banks_gpu.py).
"""
import numpy as np


def exact_analysis(U, responses, s):
    """Every filter applied exactly: column i of the result is U diag(responses[i]) U^T s.
    ``responses`` is (Nf, N), the filters' values at the eigenvalues; returns (N, Nf)."""
    s_hat = U.T @ np.asarray(s, dtype=np.float64)
    return U @ (responses.T * s_hat[:, None])


def gabor_responses(e, kernel):
    """Filter i of Gabor(G, g) is g translated to e_i: (Nf, N) responses g(e_l - e_i)."""
    e = np.asarray(e, dtype=np.float64)
    return np.stack([np.asarray(kernel(e - ei), dtype=np.float64).reshape(-1) for ei in e])


def gabor(e, U, kernel, s):
    """Gabor(G, g).filter(s): exact analysis by the translated kernels, (N, N)."""
    return exact_analysis(U, gabor_responses(e, kernel), s)


def modulation_table(e, U, g_e):
    """Modulation's coefficients: entry (l, i) is filter i's response at e_l,
    sqrt(N) sum_v U[v, l] U[v, i] w[v] with the window w = U g(e) (modulation.py:146-162)."""
    n = U.shape[0]
    w = U @ np.asarray(g_e, dtype=np.float64)
    return np.sqrt(n) * (U.T @ (U * w[:, None]))


def modulation_first(e, U, g_e, s):
    """Modulation(G, g, modulation_first=True).filter(s): the exact filter whose responses are
    looked up in the table (the first equal eigenvalue for a repeated one)."""
    e = np.asarray(e, dtype=np.float64)
    first = np.searchsorted(e, e, side="left")
    return exact_analysis(U, modulation_table(e, U, g_e)[first].T, s)


def windowed_gft(U, windows, s):
    """Modulation(G, g).filter(s): row i is sqrt(N) U^T (s * w_i) for the window w_i, column i
    of ``windows`` (the reference's g.localize(i), sqrt(N) g(L) delta_i); (N, N)."""
    n = U.shape[0]
    s = np.asarray(s, dtype=np.float64)
    return np.stack([np.sqrt(n) * (U.T @ (s * windows[:, i])) for i in range(n)])
