"""Graph differential operator on the device: edge list, incidence matrix D, grad, div.

Mirror of ``pygsp/graphs/difference.py`` (:9-331) -- ``D``, ``compute_differential_operator``,
``grad``, ``div`` -- and of ``Graph.get_edge_list`` (graph.py:962-1029) and
``Graph.dirichlet_energy`` (graph.py:642-702), mixed into :class:`Graph`.  Same names,
arguments, exceptions and log messages.

``G.D`` is a :class:`DeviceCSR` of shape (N, Ne) built in HBM from W by csrc/difference.cu;
``G.D.T`` is D^T (Ne, N), built with it (its arrays are the CSC arrays of the reference's D:
``G.D.to_scipy_csc()`` gives the reference's ``csc_matrix``).  A self-loop is an edge whose
column of D is empty: the reference's two entries of a loop cancel and ``eliminate_zeros``
drops them.  ``grad`` and ``div`` are the SpMM kernel on D^T and D; ``dirichlet_energy`` is
``L x`` followed by the float64 Gram kernel for x^T (L x).  NumPy in -> NumPy out (graph
dtype), CUDA tensor in -> CUDA tensor out; inputs are never modified.
"""
import numpy as np

from .. import _native as nat
from .csr import DeviceCSR

_LAP = {"combinatorial": 0, "normalized": 1}


class DifferenceMixIn:

    @property
    def D(self):
        r"""Differential operator (for gradient and divergence), a :class:`DeviceCSR` (N, Ne).

        Is computed by :func:`compute_differential_operator`.
        """
        if self._D is None:
            self.logger.warning("The differential operator G.D is not "
                                "available, we need to compute it. Explicitly "
                                "call G.compute_differential_operator() "
                                "once beforehand to suppress the warning.")
            self.compute_differential_operator()
        return self._D

    def _edges_device(self):
        """(eptr, sources, targets, weights, Dt indptr) on the device, in CSR order."""
        torch = nat.require_cuda()
        W, n, ne = self._adjacency, self.n_vertices, self.n_edges
        if self.is_directed():
            eptr = W.indptr
        else:
            eptr = torch.empty(n + 1, dtype=torch.int32, device=self.device)
            with torch.cuda.device(self.device):
                nat.call("gsp_edge_offsets", nat.i64(n), W.indptr, W.indices, eptr,
                         self._stream())
        sources = torch.empty(ne, dtype=torch.int32, device=self.device)
        targets = torch.empty(ne, dtype=torch.int32, device=self.device)
        weights = torch.empty(ne, dtype=self.dtype, device=self.device)
        dt_indptr = torch.empty(ne + 1, dtype=torch.int32, device=self.device)
        self._call("gsp_edge_list", nat.i64(n), nat.i64(ne), W.indptr, W.indices, W.data, eptr,
                   sources, targets, weights, dt_indptr)
        return eptr, sources, targets, weights, dt_indptr

    def get_edge_list(self):
        r"""Return an edge list, an alternative representation of the graph (graph.py:962-1029).

        ``(sources, targets, weights)`` as NumPy arrays (int32, int32, graph dtype) of length
        ``G.n_edges``: the upper triangle of W (self-loops included) for an undirected graph,
        every stored entry for a directed one, in row-major order (``sparse.triu(W,
        format='coo')`` / ``W.tocoo()``).
        """
        _, sources, targets, weights, _ = self._edges_device()
        sources, targets, weights = (t.cpu().numpy() for t in (sources, targets, weights))
        assert self.n_edges == sources.size == targets.size == weights.size
        return sources, targets, weights

    def compute_differential_operator(self):
        r"""Compute the graph differential operator D, with L = D D^T (cached).

        difference.py:26-166.  Built on the device from W (and W^T for a directed graph):
        D[s, k] = -sqrt(w), D[t, k] = +sqrt(w) for the combinatorial Laplacian,
        -sqrt(w / dw[s]) and +sqrt(w / dw[t]) for the normalized one, both divided by sqrt(2)
        for a directed graph; computed in float64 and rounded once to the graph's dtype.
        Raises ``ValueError`` if D would hold 2^31 entries or more.
        """
        torch = nat.require_cuda()
        if self.lap_type not in _LAP:
            raise ValueError("Unknown lap_type {}".format(self.lap_type))
        W, n, ne = self._adjacency, self.n_vertices, self.n_edges
        nnz = 2 * (ne - self._n_loops)
        if nnz >= 2 ** 31:
            raise ValueError("The differential operator would have {} entries; at most 2^31 - 1 "
                             "are supported.".format(nnz))
        directed = self.is_directed()
        Wt = self._transpose() if directed else None
        dw = self._degrees()[0]
        lap = nat.i32(_LAP[self.lap_type])
        eptr, sources, targets, weights, dt_indptr = self._edges_device()

        dt_indices = torch.empty(nnz, dtype=torch.int32, device=self.device)
        dt_data = torch.empty(nnz, dtype=self.dtype, device=self.device)
        self._call("gsp_incidence_t_fill", nat.i64(ne), sources, targets, weights, dw, lap,
                   nat.i32(directed), dt_indptr, dt_indices, dt_data)

        t = (Wt.indptr, Wt.indices, Wt.data) if directed else (None, None, None)
        D = DeviceCSR.from_counts(
            (n, ne), self.dtype, self.device,
            lambda st, ip, total: nat.call("gsp_incidence_count", nat.i64(n), W.indptr, W.indices,
                                           *t[:2], ip, total, st),
            lambda st, ip, ix, d: nat.call("gsp_incidence_fill_" + self._sfx, nat.i64(n), lap,
                                           W.indptr, W.indices, W.data, eptr, *t, dw, ip, ix, d,
                                           st),
            "differential operator", nnz=nnz)
        D.T = DeviceCSR(dt_indptr, dt_indices, dt_data, (ne, n))
        self._D = D

    def grad(self, x):
        r"""Gradient D^T x of a signal on the vertices (difference.py:168-244).

        ``x``: (N,) or (N, Nsig); returns (Ne,) or (Ne, Nsig).
        """
        x = self._check_signal(x)
        return self.D.T.dot(x)

    def div(self, y):
        r"""Divergence D y of a signal on the edges (difference.py:246-331).

        ``y``: (Ne,) or (Ne, Nsig); returns (N,) or (N, Nsig).
        """
        torch = nat.require_cuda()
        if not torch.is_tensor(y):
            y = np.asanyarray(y)
        if y.shape[0] != self.Ne:
            raise ValueError("First dimension must be the number of edges "
                             "G.Ne = {}, got {}.".format(self.Ne, tuple(y.shape)))
        return self.D.dot(y)

    def dirichlet_energy(self, x):
        r"""Dirichlet energy x^T L x of a signal on the vertices (graph.py:642-702).

        A float64 scalar for an (N,) signal, the (Nsig, Nsig) float64 matrix x^T L x for an
        (N, Nsig) block: NumPy for host input, a CUDA tensor for CUDA input.  L x is the
        Laplacian's product in the graph's dtype; x^T (L x) accumulates in float64 in a fixed
        order (csrc/block.cu).
        """
        from ..filters import approximations as apx
        from .fourier import block_gram
        x = self._check_signal(x)
        xd, one_d, kind = apx._as_device_block(apx._GraphView(self.L), x)
        E = apx._leave_device(block_gram(xd, self.L.dot(xd)), kind)
        return E[0, 0] if one_d else E
