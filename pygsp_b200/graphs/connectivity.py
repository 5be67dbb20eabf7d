"""Graph connectivity on the device: is_connected, extract_components, subgraph.

Mirror of the structural half of ``pygsp.graphs.Graph`` -- ``set_signal`` (graph.py:192-216),
``subgraph`` (:218-255), ``is_weighted`` (:257-292), ``is_connected`` (:294-366) and
``extract_components`` (:444-508) -- mixed into :class:`Graph`.  Same names, arguments,
exceptions and log messages.

The reference walks the graph with a Python BFS over ``W[v].nonzero()``; here csrc/connectivity.cu
does the work in HBM:

* ``is_connected`` of an undirected graph counts the components of a union-find over the stored
  entries; of a directed graph it runs a frontier BFS from vertex 0 through W and through W^T
  (strong connectivity), a bounded batch of levels per call, reading one small state block per
  batch.
* ``subgraph`` builds ``W[vertices, :][:, vertices]`` by count -> scan -> fill through a
  multiplicity map of the kept vertices; rows come out sorted when ``vertices`` is strictly
  increasing, otherwise they are sorted by ``DeviceCSR.from_coo`` (graphs/csr.py).
* ``extract_components`` labels the components of ``W > 0`` (a negative edge does not join two
  components, as in the reference), orders the vertices by (component, id) and builds ONE
  block-diagonal CSR; component k is a slice of it.  Only the vertex ids of ``orig_idx`` and
  the component boundaries come back to the host.

Two differences from the reference: ``info['orig_idx']`` is a NumPy int64 array (the reference
stores a sorted list of the same ids), and a subgraph keeps its parent's ``dtype`` and
``device``.
"""
import numpy as np

from .. import _native as nat
from .csr import DeviceCSR

# levels of the directed BFS per launch batch: the first batch, and the cap of the doubling
_REACH_FIRST, _REACH_MAX = 8, 1024


class ConnectivityMixIn:

    def set_signal(self, signal, name):
        r"""Attach a signal to the graph (graph.py:192-216); it lands in :attr:`signals`."""
        signal = self._check_signal(signal)
        self.signals[name] = signal

    def is_weighted(self):
        r"""True unless every stored weight of W equals 1 (graph.py:257-292)."""
        torch = nat.require_cuda()
        flag = torch.empty(1, dtype=torch.int32, device=self.device)
        self._call("gsp_weights_not_one", nat.i64(self._adjacency.nnz), self._adjacency.data,
                   flag)
        return bool(flag.item())

    # ----------------------------------------------------------------- connectivity
    def is_connected(self):
        r"""Check if the graph is connected (cached; graph.py:294-366).

        An edge is any stored entry of W, negative weights included.  Undirected: every vertex is
        reachable from vertex 0 (one component).  Directed: every vertex is reachable from 0
        through W and through W^T, i.e. the graph is strongly connected.  A graph without
        vertices raises ``IndexError``, as in the reference.
        """
        if self._connected is not None:
            return self._connected
        if self.n_vertices == 0:
            raise IndexError("index 0 is out of bounds for axis 0 with size 0")
        if self.is_directed():
            self._connected = (self._reaches_all(self._adjacency)
                               and self._reaches_all(self._transpose()))
        else:
            _, n_components = self._component_labels(positive_only=False)
            self._connected = int(n_components.item()) == 1
        return self._connected

    def _component_labels(self, positive_only):
        """(labels, number of components) on the device: labels[v] = smallest vertex id of v's
        component, over the stored entries of W, or over those with weight > 0."""
        torch = nat.require_cuda()
        W, n = self._adjacency, self.n_vertices
        labels = torch.empty(n, dtype=torch.int32, device=self.device)
        n_components = torch.empty(1, dtype=torch.int64, device=self.device)
        self._call("gsp_cc_labels", nat.i64(n), W.indptr, W.indices, W.data,
                   nat.i32(positive_only), labels, n_components)
        return labels, n_components

    def _reaches_all(self, A):
        """True iff the BFS from vertex 0 over the stored entries of A reaches every vertex."""
        torch = nat.require_cuda()
        n = self.n_vertices
        visited = torch.empty(n, dtype=torch.int32, device=self.device)
        queue = torch.empty(2 * n, dtype=torch.int32, device=self.device)
        state = torch.empty(4, dtype=torch.int64, device=self.device)
        with torch.cuda.device(self.device):
            nat.call("gsp_reach_init", nat.i64(n), nat.i32(0), visited, queue, state,
                     self._stream())
            level, batch = 0, _REACH_FIRST
            while True:
                nat.call("gsp_reach_levels", nat.i64(n), A.indptr, A.indices, visited, queue,
                         state, nat.i64(level), nat.i32(batch), self._stream())
                level += batch
                s = state.cpu().numpy()
                frontier, reached = int(s[level % 3]), int(s[3])
                if frontier == 0 or reached + frontier == n:
                    return reached + frontier == n
                batch = min(2 * batch, _REACH_MAX)

    # --------------------------------------------------------------------- subgraphs
    def _vertex_ids(self, vertices):
        """(host int64 ids or None, device int32 ids) of an index list or a boolean mask:
        negative indices count from the end, out-of-range ones raise ``IndexError``."""
        torch = nat.require_cuda()
        n = self.n_vertices
        if torch.is_tensor(vertices):
            v = vertices.to(self.device)
            if v.dtype == torch.bool:
                if tuple(v.shape) != (n,):
                    raise IndexError("boolean index of shape {} for {} vertices".format(
                        tuple(v.shape), n))
                v = torch.nonzero(v).flatten()
            elif v.is_floating_point() or v.is_complex():
                raise IndexError("only integers and boolean masks are valid vertex indices")
            if v.dim() != 1:
                raise IndexError("vertex indices must be one-dimensional")
            v = v.long()
            v = torch.where(v < 0, v + n, v)
            if v.numel() and (int(v.min()) < 0 or int(v.max()) >= n):
                raise IndexError("vertex index out of range for {} vertices".format(n))
            return None, v.to(torch.int32).contiguous()
        a = np.asarray(vertices)
        if a.dtype == bool:
            if a.shape != (n,):
                raise IndexError("boolean index of shape {} for {} vertices".format(a.shape, n))
            a = np.flatnonzero(a)
        elif a.size == 0:
            a = a.reshape(0)
        elif not np.issubdtype(a.dtype, np.integer):
            raise IndexError("only integers and boolean masks are valid vertex indices")
        if a.ndim != 1:
            raise IndexError("vertex indices must be one-dimensional")
        a = a.astype(np.int64)
        a = np.where(a < 0, a + n, a)
        if a.size and (a.min() < 0 or a.max() >= n):
            bad = a[(a < 0) | (a >= n)][0]
            raise IndexError("vertex index {} is out of range for {} vertices".format(
                bad - n if bad < 0 else bad, n))
        return a, torch.from_numpy(a.astype(np.int32)).to(self.device)

    def _child(self, W, ids_host, ids_dev):
        """Graph on W with the coords, plotting, Laplacian type and signals of the vertices
        ids of this graph (graph.py:248-255), in this graph's dtype and on its device."""
        from .graph import Graph
        torch = nat.require_cuda()

        def host_ids():
            return ids_host if ids_host is not None else ids_dev.cpu().numpy().astype(np.int64)
        coords = self.coords[host_ids()] if hasattr(self, "coords") else None
        graph = Graph(W, self.lap_type, coords, self.plotting, dtype=self.dtype,
                      device=self.device)
        for name, signal in self.signals.items():
            if torch.is_tensor(signal):
                graph.set_signal(signal[ids_dev.to(signal.device).long()], name)
            else:
                graph.set_signal(signal[host_ids()], name)
        return graph

    def subgraph(self, vertices):
        r"""Create a subgraph from a list of vertices (graph.py:218-255).

        ``vertices``: a list (or array, or tensor) of indices -- unsorted, repeated and negative
        indices allowed -- or a boolean mask of length N.  The result is a :class:`Graph` on
        ``W[vertices, :][:, vertices]`` with the same ``lap_type``, ``plotting``,
        ``coords[vertices]`` and every signal sliced the same way (NumPy signals stay NumPy,
        CUDA tensors stay on the device), in this graph's dtype and on its device.  Raises
        ``IndexError`` for an index out of range and ``ValueError`` if the subgraph would hold
        2^31 entries or more.
        """
        torch = nat.require_cuda()
        ids_host, v = self._vertex_ids(vertices)
        if ids_host is not None:
            increasing = bool(np.all(ids_host[1:] > ids_host[:-1]))
        else:
            increasing = v.numel() < 2 or bool(torch.all(v[1:] > v[:-1]))
        W, rows = self._adjacency.induced(v, None, increasing)
        if rows is not None:        # repeated or unordered vertices: sort each row
            W = DeviceCSR.from_coo(rows, W.indices, W.data, W.shape)
        return self._child(W, ids_host, v)

    def extract_components(self):
        r"""Split the graph into connected components (graph.py:444-508).

        Connectivity is the one of ``A = W > 0``: a negative edge does not join two components
        (while :meth:`is_connected` counts it).  Components come in order of their smallest
        vertex; each is ``self.subgraph(ids)`` for its sorted vertex ids, with ``info =
        {'orig_idx': ids}`` (a NumPy int64 array).  Directed graphs raise
        ``NotImplementedError``, as in the reference.
        """
        torch = nat.require_cuda()
        if self.is_directed():
            raise NotImplementedError("Directed graphs not supported yet.")
        n, dev = self.n_vertices, self.device
        if n == 0:
            return []
        labels, _ = self._component_labels(positive_only=True)
        perm = torch.empty(n, dtype=torch.int32, device=dev)
        comp_ptr = torch.empty(n + 1, dtype=torch.int32, device=dev)
        n_components = torch.empty(1, dtype=torch.int64, device=dev)
        with torch.cuda.device(dev):
            nat.call("gsp_component_order", nat.i64(n), labels, perm, comp_ptr, n_components,
                     self._stream())
        # one block-diagonal CSR: component k is rows / columns [ptr[k], ptr[k+1])
        S, _ = self._adjacency.induced(perm, labels, increasing=True)
        ptr = comp_ptr[:int(n_components.item()) + 1]
        offsets = S.indptr[ptr.long()].cpu().numpy()
        ptr = ptr.cpu().numpy()
        ids_all = perm.cpu().numpy().astype(np.int64)
        graphs = []
        for k in range(len(ptr) - 1):
            a, b, e0, e1 = int(ptr[k]), int(ptr[k + 1]), int(offsets[k]), int(offsets[k + 1])
            self.logger.info("Constructing subgraph for component of size {}.".format(b - a))
            W = DeviceCSR(S.indptr[a:b + 1] - e0, S.indices[e0:e1] - a, S.data[e0:e1],
                          (b - a, b - a))
            ids = ids_all[a:b]
            graph = self._child(W, ids, perm[a:b])
            graph.info = {"orig_idx": ids}
            graphs.append(graph)
        return graphs
