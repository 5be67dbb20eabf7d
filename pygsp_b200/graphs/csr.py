"""CSR matrix resident in HBM: int32 indptr / indices + float32|float64 data.

This is what ``Graph.W`` and ``Graph.L`` are in this engine (the reference
holds ``scipy.sparse.csr_matrix`` objects, graph.py:109,620).  Besides the
read-only surface of the filtering path (``shape``, ``nnz``, ``dot``,
``toarray``, ``diagonal``, ``to_scipy``), this module owns every device
operation that builds or reshapes CSR structure: assembly from COO triplets
(``from_coo``), ``transpose``, ``symmetrize``, ``eliminate_zeros``, induced
submatrices (``induced``), the row id of every entry (:func:`row_ids`) and
the dense float64 copy (``to_dense``).  The differential operator ``G.D`` is
one too, (N, Ne), with its transpose attached as ``.T`` by the builder
(graphs/difference.py).
"""
import numpy as np

from .. import _native as nat

_SYMMETRIZE_MODES = {"maximum": 0, "fill": 1, "tril": 2, "triu": 3}


def row_ids(indptr):
    """Row id (int64) of every entry of the CSR structure ``indptr``, on its device."""
    import torch
    counts = (indptr[1:] - indptr[:-1]).long()
    return torch.repeat_interleave(torch.arange(indptr.numel() - 1, device=indptr.device), counts)


def index32(ids, n, device):
    """Contiguous int32 copy of integer ids on ``device``.  int64 ids outside [0, n) become -1,
    which the range checks of the kernels refuse; a plain cast would wrap 2^32 + k onto k."""
    import torch
    ids = ids.to(device)
    if ids.dtype == torch.int64:
        ids = torch.where((ids >= 0) & (ids < n), ids, -1)
    return ids.to(torch.int32).contiguous()


class DeviceCSR:
    def __init__(self, indptr, indices, data, shape):
        self.indptr = indptr
        self.indices = indices
        self.data = data
        self.shape = (int(shape[0]), int(shape[1]))
        self._plans = {}

    def tile_plan(self, nsig, nscales):
        """Tiling of the float32 TMA path for this matrix (cached; None = row-group kernel)."""
        torch = nat.require_cuda()
        if self.data.dtype != torch.float32:
            return None
        key = (int(nsig), int(nscales))
        if key not in self._plans:
            plan = nat.TilePlan()
            with torch.cuda.device(self.device):
                nat.call("gsp_cheby_tile_plan", nat.i64(self.shape[0]), self.indptr,
                         nat.i64(nsig), nat.i32(nscales), plan, nat.stream_ptr(self.device))
            self._plans[key] = plan if plan.rows_per_tile > 0 else None
        return self._plans[key]

    def pair_plan(self, rows_per_tile):
        """Slot tables of the paired Clenshaw launch for this matrix (cached): the device tensors
        (slots_fwd, slots_rev, nbr_ptr, nbr_idx) of ``gsp_cheby_pair_plan_host``, which runs on a
        host copy of the structure.  GSPB200_PAIR_LAG overrides the lag (a probe)."""
        import ctypes
        import os
        torch = nat.require_cuda()
        lag = int(os.environ.get("GSPB200_PAIR_LAG") or 192)
        key = ("pairs", int(rows_per_tile), lag)
        if key not in self._plans:
            indptr = self.indptr.cpu().numpy()
            indices = self.indices.cpu().numpy()
            n, T = self.shape[0], self.shape[0] // int(rows_per_tile)
            count = ctypes.c_int64(0)
            cap = 16 * T
            while True:
                nbr_ptr = np.empty(T + 1, dtype=np.int32)
                nbr_idx = np.empty(cap, dtype=np.int32)
                fwd = np.empty(2 * T, dtype=np.int32)
                rev = np.empty(2 * T, dtype=np.int32)
                nat.call("gsp_cheby_pair_plan_host", nat.i64(n), indptr, indices,
                         nat.i32(rows_per_tile), nat.i32(lag), nat.i64(cap), nbr_ptr, nbr_idx,
                         fwd, rev, ctypes.byref(count))
                if count.value <= cap:
                    break
                cap = count.value
            self._plans[key] = tuple(torch.from_numpy(a).to(self.device)
                                     for a in (fwd, rev, nbr_ptr, nbr_idx[:max(count.value, 1)]))
        return self._plans[key]

    def ring_plan(self, rows_per_tile):
        """Neighbour rings of the tiled Clenshaw steps for this matrix (cached): a
        ``_native.RingPlan`` whose device tables are those of ``gsp_cheby_ring_plan_host``,
        which runs on a host copy of the structure.  ``ring_max`` is the largest ring; whether
        it fits a step of ``nsig`` signals is ``gsp_cheby_ring_fits``.  None when the largest
        ring exceeds the 16-bit ring positions."""
        import ctypes
        torch = nat.require_cuda()
        key = ("rings", int(rows_per_tile))
        if key not in self._plans:
            indptr = self.indptr.cpu().numpy()
            indices = self.indices.cpu().numpy()
            n, T = self.shape[0], self.shape[0] // int(rows_per_tile)
            count, ring_max = ctypes.c_int64(0), ctypes.c_int32(0)
            cap = 32 * T
            while True:
                meta = np.empty(4 * T, dtype=np.int32)
                runs = np.empty(2 * cap, dtype=np.int32)
                local = np.empty(max(len(indices), 1), dtype=np.uint16)
                nat.call("gsp_cheby_ring_plan_host", nat.i64(n), indptr, indices,
                         nat.i32(rows_per_tile), nat.i64(cap), meta, runs, local,
                         ctypes.byref(count), ctypes.byref(ring_max))
                if count.value <= cap or ring_max.value > 65535:
                    break
                cap = count.value
            plan = None
            if ring_max.value <= 65535:
                plan = nat.RingPlan(int(rows_per_tile), ring_max.value)
                plan.tensors = tuple(torch.from_numpy(a).to(self.device)
                                     for a in (meta, runs[:2 * max(count.value, 1)],
                                               local.view(np.int16)))
                plan.tile_meta, plan.runs, plan.local = (t.data_ptr() for t in plan.tensors)
            self._plans[key] = plan
        return self._plans[key]

    # -- construction ---------------------------------------------------------
    @classmethod
    def from_scipy(cls, M, dtype, device):
        torch = nat.require_cuda()
        M = M.tocsr()
        if M.nnz >= 2 ** 31:
            raise ValueError("nnz must fit int32 indices")
        indptr = torch.from_numpy(np.ascontiguousarray(M.indptr, dtype=np.int32)).to(device)
        indices = torch.from_numpy(np.ascontiguousarray(M.indices, dtype=np.int32)).to(device)
        data = torch.from_numpy(np.ascontiguousarray(M.data)).to(device=device, dtype=dtype)
        return cls(indptr, indices, data, M.shape)

    @classmethod
    def from_coo(cls, rows, cols, vals, shape):
        """Canonical CSR of COO triplets in HBM: what ``sparse.csr_matrix(coo)`` does at
        graph.py:109 -- sort by (row, col), sum duplicates -- on the device
        (``gsp_coo_to_csr_*``).  The values of one (row, col) are added one after the other in
        the order they are given, in the value type, starting from the first (the arithmetic of
        a sequential ``sum_duplicates``), so the result is reproducible bit for bit.  Integer
        rows / cols, float32 or float64 vals; the result lives on vals' device.  An index
        outside [0, n) raises ``NativeError``, int64 ones included (they are not cast to int32
        first).  ``ValueError`` for 2^31 triplets or more, before anything is touched."""
        nnz = int(vals.numel())
        if nnz >= 2 ** 31:
            raise ValueError("The result would have {} entries; at most 2^31 - 1 are "
                             "supported.".format(nnz))
        import ctypes
        torch = nat.require_cuda()
        dev, n = vals.device, int(shape[0])
        indptr = torch.empty(n + 1, dtype=torch.int32, device=dev)
        indices = torch.empty(nnz, dtype=torch.int32, device=dev)
        data = torch.empty(nnz, dtype=vals.dtype, device=dev)
        uniq = ctypes.c_int64(0)
        with torch.cuda.device(dev):
            nat.call("gsp_coo_to_csr_" + nat.suffix(vals.dtype), nat.i64(n), nat.i64(nnz),
                     index32(rows, n, dev), index32(cols, int(shape[1]), dev),
                     vals.contiguous(), indptr, indices, data, ctypes.byref(uniq),
                     nat.stream_ptr(dev))
        m = int(uniq.value)
        return cls(indptr, indices[:m].contiguous(), data[:m].contiguous(), shape)

    def _call(self, name, *args):
        """Native entry point ``name`` on this matrix's device and its current stream."""
        torch = nat.require_cuda()
        with torch.cuda.device(self.device):
            nat.call(name, *args, nat.stream_ptr(self.device))

    def _empty(self, nnz):
        """(indices, data) buffers of nnz entries on this matrix's device and in its dtype."""
        torch = nat.require_cuda()
        return (torch.empty(nnz, dtype=torch.int32, device=self.device),
                torch.empty(nnz, dtype=self.dtype, device=self.device))

    # -- reshaping ------------------------------------------------------------------
    def transpose(self):
        """M^T of a square matrix as sorted CSR (``gsp_csr_transpose_*``)."""
        torch = nat.require_cuda()
        n = self.shape[0]
        tp = torch.empty(n + 1, dtype=torch.int32, device=self.device)
        ti, td = self._empty(self.nnz)
        self._call("gsp_csr_transpose_" + nat.suffix(self.dtype), nat.i64(n), nat.i64(self.nnz),
                   self.indptr, self.indices, self.data, tp, ti, td)
        return DeviceCSR(tp, ti, td, self.shape)

    def symmetrize(self, method="average", transpose=None):
        """utils.symmetrize(M, method) of a square matrix, on the device (utils.py:244-277).

        Each row of M is merged with the same row of M^T (``transpose``, when the caller has it
        already): 'average' is (M + M^T)/2 (``gsp_csr_average_*``); 'maximum', 'fill', 'tril' and
        'triu' go through ``gsp_csr_symmetrize_*``.  The reference's arithmetic, so values are
        bit-equal to SciPy's in float64.  Exact zeros are dropped."""
        if self.shape[0] != self.shape[1]:
            raise ValueError("Matrix must be square.")
        if method == "average":
            name, mode = "gsp_csr_average_", ()
        elif method in _SYMMETRIZE_MODES:
            name, mode = "gsp_csr_symmetrize_", (nat.i32(_SYMMETRIZE_MODES[method]),)
        else:
            raise ValueError("Unknown symmetrization method {}.".format(method))
        torch = nat.require_cuda()
        n, sfx = self.shape[0], nat.suffix(self.dtype)
        T = self.transpose() if transpose is None else transpose
        operands = (self.indptr, self.indices, self.data, T.indptr, T.indices, T.data)
        sp = torch.empty(n + 1, dtype=torch.int32, device=self.device)
        self._call(name + "count_" + sfx, nat.i64(n), *mode, *operands, sp)
        si, sd = self._empty(int(sp[-1].item()) if n else 0)
        self._call(name + "fill_" + sfx, nat.i64(n), *mode, *operands, sp, si, sd)
        return DeviceCSR(sp, si, sd, self.shape)

    def eliminate_zeros(self):
        """M without its stored zeros (graph.py:128), by the compaction kernels."""
        torch = nat.require_cuda()
        n, sfx = self.shape[0], nat.suffix(self.dtype)
        indptr = torch.empty(n + 1, dtype=torch.int32, device=self.device)
        self._call("gsp_csr_compact_count_" + sfx, nat.i64(n), self.indptr, self.data, indptr)
        indices, data = self._empty(int(indptr[-1].item()) if n else 0)
        self._call("gsp_csr_compact_fill_" + sfx, nat.i64(n), self.indptr, self.indices, self.data,
                   indptr, indices, data)
        return DeviceCSR(indptr, indices, data, self.shape)

    def induced(self, v, labels=None, increasing=False):
        """Entries of M[v, :][:, v] (m x m) for device int32 ids v, by map -> count -> fill.

        With ``labels`` (int32, one per vertex of M) only the entries whose two ends carry the
        same label are kept.  Returns (S, rows).  ``increasing`` (v strictly increasing, or
        listing the vertices by (label, id) with labels given): the rows come out sorted, S is
        canonical and rows is None.  Otherwise each row of S holds its entries in M's column order
        mapped through v, unsorted, and rows (int32) is the row of every entry, so that
        ``DeviceCSR.from_coo(rows, S.indices, S.data, S.shape)`` is the canonical matrix.
        ``ValueError`` when the result would hold 2^31 entries or more."""
        torch = nat.require_cuda()
        n, m, dev = self.shape[0], int(v.numel()), self.device
        if m == 0:
            S = DeviceCSR(torch.zeros(1, dtype=torch.int32, device=dev), *self._empty(0), (0, 0))
            return S, None if increasing else S.indices
        mptr = torch.empty(n + 1, dtype=torch.int32, device=dev)
        mpos = torch.empty(m, dtype=torch.int32, device=dev)
        s_indptr = torch.empty(m + 1, dtype=torch.int32, device=dev)
        nnz = torch.empty(1, dtype=torch.int64, device=dev)
        self._call("gsp_vertex_map", nat.i64(n), nat.i64(m), v, mptr, mpos)
        self._call("gsp_subgraph_count", nat.i64(m), self.indptr, self.indices, v, mptr, labels,
                   s_indptr, nnz)
        nnz = int(nnz.item())
        if nnz >= 2 ** 31:
            raise ValueError("The subgraph would have {} entries; at most 2^31 - 1 are "
                             "supported.".format(nnz))
        s_indices, s_data = self._empty(nnz)
        rows = None if increasing else torch.empty(nnz, dtype=torch.int32, device=dev)
        self._call("gsp_subgraph_fill_" + nat.suffix(self.dtype), nat.i64(m), self.indptr,
                   self.indices, self.data, v, mptr, mpos, labels, s_indptr, s_indices, s_data,
                   rows)
        return DeviceCSR(s_indptr, s_indices, s_data, (m, m)), rows

    # -- introspection --------------------------------------------------------
    @property
    def nnz(self):
        return int(self.indices.numel())

    @property
    def dtype(self):
        return self.data.dtype

    @property
    def device(self):
        return self.data.device

    def __repr__(self):
        return "<DeviceCSR {}x{}, nnz={}, {}, {}>".format(
            self.shape[0], self.shape[1], self.nnz, self.data.dtype, self.data.device)

    # -- leaving the device, dense copies ----------------------------------------
    def to_scipy(self):
        from scipy import sparse
        return sparse.csr_matrix((self.data.cpu().numpy(), self.indices.cpu().numpy(),
                                  self.indptr.cpu().numpy()), shape=self.shape)

    def to_scipy_csc(self):
        """The matrix as ``scipy.sparse.csc_matrix``, for a matrix whose builder set ``.T``
        (the differential operator: its CSC arrays are the CSR arrays of its transpose)."""
        from scipy import sparse
        T = getattr(self, "T", None)
        if T is None:
            raise AttributeError("to_scipy_csc needs the transpose built with the matrix (.T)")
        return sparse.csc_matrix((T.data.cpu().numpy(), T.indices.cpu().numpy(),
                                  T.indptr.cpu().numpy()), shape=self.shape)

    def toarray(self):
        return self.to_scipy().toarray()

    def to_dense(self):
        """The matrix as a dense float64 tensor on its device."""
        torch = nat.require_cuda()
        dense = torch.zeros(self.shape, dtype=torch.float64, device=self.device)
        dense[row_ids(self.indptr), self.indices.long()] = self.data.double()
        return dense

    def diagonal(self):
        return self.to_scipy().diagonal()

    # -- product: scipy's csr_matrix.dot on the device SpMM kernel ------------------
    def dot(self, x):
        """``A @ x`` for a vector or an (n, nsig) block; numpy in -> numpy out.

        A rectangular matrix (the differential operator) always takes the SpMM kernel, which
        reads x at column indices only; the SpMV's window form assumes a square matrix.
        """
        torch = nat.require_cuda()
        host = not torch.is_tensor(x)
        xt = torch.as_tensor(np.asarray(x) if host else x).to(device=self.device, dtype=self.dtype)
        if xt.shape[0] != self.shape[1]:
            raise ValueError("dimension mismatch")
        flat = xt.reshape(xt.shape[0], int(np.prod(xt.shape[1:]))).contiguous()
        square = self.shape[0] == self.shape[1]
        if not square and (flat.numel() == 0 or self.shape[0] == 0):
            y = torch.zeros((self.shape[0], flat.shape[1]), dtype=self.dtype, device=self.device)
            y = y.reshape((self.shape[0],) + tuple(xt.shape[1:]))
            return y.cpu().numpy() if host else y
        y = torch.empty((self.shape[0], flat.shape[1]), dtype=self.dtype, device=self.device)
        with torch.cuda.device(self.device):
            if flat.shape[1] == 1 and square:          # one vector: the sub-warp SpMV
                nat.call("gsp_spmv_" + nat.suffix(self.dtype), nat.i64(self.shape[0]),
                         nat.i64(self.nnz), self.indptr, self.indices, self.data, flat, y,
                         nat.stream_ptr(self.device))
            else:
                nat.call("gsp_spmm_" + nat.suffix(self.dtype), nat.i64(self.shape[0]),
                         self.indptr, self.indices, self.data, flat, nat.i64(flat.shape[1]), y,
                         nat.stream_ptr(self.device))
        y = y.reshape((self.shape[0],) + tuple(xt.shape[1:]))
        return y.cpu().numpy() if host else y

    __matmul__ = dot
