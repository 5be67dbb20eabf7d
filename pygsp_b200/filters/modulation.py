"""Modulation filter bank, the windowed graph Fourier transform (mirror of
pygsp/filters/modulation.py:99-177)."""
import numpy as np

from .. import _native as nat
from .filter import Filter
from .gabor import check_mother_kernel


class Modulation(Filter):
    r"""The mother kernel localised by graph modulation: one filter per vertex.

    ``modulation_first=False`` (default): :meth:`filter` is the windowed graph Fourier transform,
    ``Y[i] = sqrt(N) U^T (s * w_i)`` with the window ``w_i = sqrt(N) g(L) delta_i`` (the kernel's
    :meth:`localize`, Chebyshev order 30), all N windows formed as one block ``sqrt(N) g(L) I``.
    Unlike the reference's loop of N calls, ``s`` must be one signal (1-D): any other shape raises
    ``ValueError``.

    ``modulation_first=True``: :meth:`filter` is the exact filter of the bank.  Filter i has the
    response ``c[l, i] = sqrt(N) sum_v U[v, l] U[v, i] (U g(e))[v]`` at the eigenvalue ``e_l``;
    :meth:`evaluate` looks these up at the eigenvalues and returns NaN at any other frequency.
    Both need the full Fourier basis.
    """

    def __init__(self, graph, kernel, modulation_first=False):
        check_mother_kernel(graph, kernel)
        self.G = graph
        self._kernels = kernel
        self._modulation_first = modulation_first
        self.n_features_in, self.n_features_out = 1, graph.N
        self.n_filters = self.Nf = graph.N
        self.shape = (graph.N, 1)
        self.fused_synthesis = True
        self.clenshaw = True

    def _coefficient_table(self):
        """(N, N) host float64: row l holds every filter's response at e_l."""
        if not hasattr(self, "_coefficients"):
            from ..graphs import fourier
            G = self.G
            U = G._device_basis()
            g = self._kernels.evaluate(G.e)[0]
            window = fourier.block_combine(U, g[:, None])               # U g(e): (N, 1)
            table = fourier.block_gram(U, U * window) * np.sqrt(G.N)    # U^T diag(U g(e)) U
            self._coefficients = table.cpu().numpy()
        return self._coefficients

    def evaluate(self, x):
        r"""Responses at ``x``: shape (N, *x.shape); NaN where x is not an eigenvalue (the first
        equal eigenvalue is taken for a repeated one)."""
        x = np.asanyarray(x)
        table = self._coefficient_table()
        e = np.asarray(self.G.e)
        flat = x.reshape(-1)
        pos = np.searchsorted(e, flat, side="left")
        hit = pos < e.size
        hit[hit] = e[pos[hit]] == flat[hit]
        y = np.full((self.n_features_out, flat.size), np.nan)
        y[:, hit] = table[pos[hit]].T
        return y.reshape((self.n_features_out,) + x.shape)

    def filter(self, s, method="exact", order=None):
        r"""The exact filter (``modulation_first=True``) or the windowed graph Fourier transform
        (N, N) of a 1-D signal ``s``.  ``method`` and ``order`` are ignored (modulation.py:164)."""
        if self._modulation_first:
            return super().filter(s, method="exact")
        from ..graphs import fourier
        from . import approximations as apx
        torch = nat.require_cuda()
        G, N = self.G, self.G.N
        if s.ndim != 1 or s.shape[0] != N:
            raise ValueError("The windowed graph Fourier transform takes one signal of "
                             "N = {} values, got shape {}.".format(N, tuple(s.shape)))
        L = apx._laplacian_on_device(G)
        x, _, kind = apx._as_device_block(apx._GraphView(L), s)
        eye = torch.eye(N, dtype=L.dtype, device=L.device)
        windows = self._kernels.filter(eye) * np.sqrt(N)                # column i: w_i
        Y = fourier.block_gram(G._device_basis(), x * windows) * np.sqrt(N)
        return apx._leave_device(Y.T.contiguous().to(L.dtype), kind)
