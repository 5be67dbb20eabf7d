"""CSR matrix resident in HBM: int32 indptr / indices + float32|float64 data.

This is what ``Graph.W`` and ``Graph.L`` are in this engine (the reference
holds ``scipy.sparse.csr_matrix`` objects, graph.py:109,620).  It offers the
small read-only surface the filtering path and its callers use: ``shape``,
``nnz``, ``dot``, ``toarray``, ``diagonal``, plus ``to_scipy`` to leave the
device.  The differential operator ``G.D`` is one too, (N, Ne), with its
transpose attached as ``.T`` by the builder (graphs/difference.py).
"""
import numpy as np

from .. import _native as nat


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

    # -- leaving the device -----------------------------------------------------
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
