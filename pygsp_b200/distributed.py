"""Vertex-partitioned Chebyshev filtering: one process per GPU, halo exchange per step.

The reference is single-process (SURVEY.md 8e); this is the multi-GPU scale-out of
``approximations.cheby_op`` (pygsp/filters/approximations.py:58-114).  The graph's
vertices are split into P contiguous row blocks.  Rank p owns rows
[bounds[p], bounds[p+1]) of L and the matching slices of T_{k-2}, T_{k-1} and r;
the only data a recurrence step needs from other ranks are the rows of T_{k-1}
its stored columns reference -- the *halo*.  Per step and per rank:

    boundary rows (those with a remote column)   -> fused step kernel
    pack their new values per peer, all-to-all-v -> halo of T_k      (NCCL, NVLink)
    interior rows                                -> fused step kernel, overlapped
                                                    with the exchange on a second stream

Row sums are accumulated in the stored order of the *global* CSR rows (column ids
are renamed, never re-sorted), so the partitioned result equals the single-GPU
result bit for bit.

Host-side planning is NumPy + ``torch.distributed`` (NCCL on GPUs, gloo in the CPU
tests); the compute is the same C-ABI step kernel as the single-GPU path.
"""
import numpy as np

from . import _native as nat
from .graphs.csr import row_ids


def even_bounds(n, parts):
    """Contiguous 1-D partition: bounds[p] = floor(n * p / parts)."""
    return (np.arange(parts + 1, dtype=np.int64) * n) // parts


class HaloPlan:
    """Everything rank ``rank`` needs to know about its row block, on the host.

    Parameters
    ----------
    rows : scipy.sparse.csr_matrix, shape (n_local, N)
        Rows [bounds[rank], bounds[rank+1]) of the global Laplacian with GLOBAL
        column ids, entries in the global CSR order.
    bounds : array of P + 1 ints
    rank, group : this process and its ``torch.distributed`` group (None = world)

    Attributes (all NumPy, local ids are in the *local order* below)
    ----------
    perm : local order -> original local row.  Boundary rows first (padded to a
        multiple of 4 rows with interior rows), interior rows after.
    n_boundary : rows in the first launch
    indptr, indices, data : local CSR, shape (n_local, n_local + n_halo); column
        j < n_local is local row j (local order), column n_local + h is halo slot h
    halo_ids : global ids of the halo slots, ascending (hence grouped by owner)
    recv_counts[q], send_counts[q], send_idx : the all-to-all-v of one step
    """

    def __init__(self, rows, bounds, rank, group=None, exchange_ids=None):
        bounds = np.asarray(bounds, dtype=np.int64)
        P = len(bounds) - 1
        lo, hi = int(bounds[rank]), int(bounds[rank + 1])
        rows = rows.tocsr()
        n_local = hi - lo
        if rows.shape[0] != n_local:
            raise ValueError("rows must hold exactly the rank's row block")
        self.rank, self.parts, self.bounds = rank, P, bounds
        self.n_local, self.n_global = n_local, int(bounds[-1])
        indptr = rows.indptr.astype(np.int64)
        cols = rows.indices.astype(np.int64)
        owned = (cols >= lo) & (cols < hi)

        # halo slots: distinct remote columns, ascending => contiguous per owner
        self.halo_ids = np.unique(cols[~owned])
        owner = np.searchsorted(bounds, self.halo_ids, side="right") - 1
        self.recv_counts = np.bincount(owner, minlength=P).astype(np.int64)
        self.n_halo = int(self.halo_ids.size)

        # local order: boundary rows first
        row_of = np.repeat(np.arange(n_local), np.diff(indptr))
        is_boundary = np.bincount(row_of[~owned], minlength=n_local) > 0
        boundary = np.flatnonzero(is_boundary)
        interior = np.flatnonzero(~is_boundary)
        pad = min((-boundary.size) % 4, interior.size)
        self.perm = np.concatenate([boundary, interior]).astype(np.int64)
        self.n_boundary = int(boundary.size + pad)
        self.n_true_boundary = int(boundary.size)
        inv = np.empty(n_local, dtype=np.int64)
        inv[self.perm] = np.arange(n_local)
        self.inv_perm = inv

        # local CSR: permute rows, rename columns, keep the within-row order
        counts = np.diff(indptr)[self.perm]
        new_ptr = np.zeros(n_local + 1, dtype=np.int64)
        np.cumsum(counts, out=new_ptr[1:])
        gather = np.repeat(indptr[self.perm] - new_ptr[:-1], counts) + np.arange(new_ptr[-1])
        c = cols[gather]
        mine = (c >= lo) & (c < hi)
        local = np.empty_like(c)
        local[mine] = inv[c[mine] - lo]
        local[~mine] = n_local + np.searchsorted(self.halo_ids, c[~mine])
        if new_ptr[-1] >= 2 ** 31 or n_local + self.n_halo >= 2 ** 31:
            raise ValueError("local block must fit int32 indices")
        self.indptr = new_ptr.astype(np.int32)
        self.indices = local.astype(np.int32)
        self.data = rows.data[gather]

        # who needs which of my rows: exchange the halo id lists once
        if exchange_ids is None:
            exchange_ids = _exchange_ids_torch
        requested, self.send_counts = exchange_ids(self.halo_ids, self.recv_counts, rank, P, group)
        self.send_idx = inv[requested - lo]              # local-order rows to pack, grouped by peer

    @classmethod
    def from_device(cls, indptr, indices, data, bounds, rank, group=None, exchange_ids=None):
        """The same plan from a row block that already lives in HBM (CUDA tensors ``indptr``
        (n_local + 1), ``indices`` (GLOBAL column ids), ``data``): every nnz-sized step runs as
        torch device ops and the local CSR stays on the device (``indices`` / ``data`` /
        ``indptr`` are CUDA tensors, everything row- or halo-sized is NumPy as usual).  Used by
        the graphs that are generated per rank on the GPU (bench config 5, strong scaling)."""
        import torch
        self = cls.__new__(cls)
        bounds = np.asarray(bounds, dtype=np.int64)
        P = len(bounds) - 1
        lo, hi = int(bounds[rank]), int(bounds[rank + 1])
        n_local = hi - lo
        if indptr.numel() != n_local + 1:
            raise ValueError("rows must hold exactly the rank's row block")
        dev = indices.device
        self.rank, self.parts, self.bounds = rank, P, bounds
        self.n_local, self.n_global = n_local, int(bounds[-1])
        ptr = indptr.long()
        counts = ptr[1:] - ptr[:-1]
        cols = indices.long()
        owned = (cols >= lo) & (cols < hi)
        halo_ids = torch.unique(cols[~owned])                    # sorted
        self.halo_ids = halo_ids.cpu().numpy()
        owner = np.searchsorted(bounds, self.halo_ids, side="right") - 1
        self.recv_counts = np.bincount(owner, minlength=P).astype(np.int64)
        self.n_halo = int(self.halo_ids.size)
        row_of = row_ids(indptr)
        is_boundary = torch.zeros(n_local, dtype=torch.bool, device=dev)
        is_boundary[row_of[~owned]] = True
        boundary = torch.nonzero(is_boundary).flatten()
        interior = torch.nonzero(~is_boundary).flatten()
        pad = min((-int(boundary.numel())) % 4, int(interior.numel()))
        perm = torch.cat([boundary, interior])
        self.n_boundary = int(boundary.numel()) + pad
        self.n_true_boundary = int(boundary.numel())
        inv = torch.empty(n_local, dtype=torch.int64, device=dev)
        inv[perm] = torch.arange(n_local, device=dev)
        self.perm, self.inv_perm = perm.cpu().numpy(), inv.cpu().numpy()
        del row_of, is_boundary
        new_counts = counts[perm]
        new_ptr = torch.zeros(n_local + 1, dtype=torch.int64, device=dev)
        torch.cumsum(new_counts, 0, out=new_ptr[1:])
        nnz = int(new_ptr[-1].item())
        if nnz >= 2 ** 31 or n_local + self.n_halo >= 2 ** 31:
            raise ValueError("local block must fit int32 indices")
        gather = torch.repeat_interleave(ptr[:-1][perm] - new_ptr[:-1], new_counts) + \
            torch.arange(nnz, device=dev)
        c = cols[gather]
        del cols, owned
        mine = (c >= lo) & (c < hi)
        local = torch.where(mine, inv[(c - lo).clamp_(0, max(n_local - 1, 0))],
                            n_local + torch.searchsorted(halo_ids, c))
        self.indptr = new_ptr.int()
        self.indices = local.int()
        self.data = data[gather]
        del gather, c, mine, local
        if exchange_ids is None:
            exchange_ids = _exchange_ids_torch
        requested, self.send_counts = exchange_ids(self.halo_ids, self.recv_counts, rank, P, group)
        self.send_idx = self.inv_perm[requested - lo]
        return self

    @property
    def nnz(self):
        return int(self.indices.numel() if hasattr(self.indices, "numel") else self.indices.size)


def _exchange_ids_torch(halo_ids, recv_counts, rank, P, group):
    """All-to-all-v of the id lists: I tell owner q which of its rows I need."""
    import torch
    import torch.distributed as dist
    if P == 1:
        return np.zeros(0, dtype=np.int64), np.zeros(1, dtype=np.int64)
    dev = torch.device("cuda", torch.cuda.current_device()) if dist.get_backend(group) == "nccl" \
        else torch.device("cpu")
    mine = torch.from_numpy(recv_counts.copy()).to(dev)
    theirs = torch.empty_like(mine)
    dist.all_to_all_single(theirs, mine, group=group)
    send_counts = theirs.cpu().numpy().astype(np.int64)
    out = torch.empty(int(send_counts.sum()), dtype=torch.int64, device=dev)
    dist.all_to_all_single(out, torch.from_numpy(halo_ids.copy()).to(dev),
                           output_split_sizes=send_counts.tolist(),
                           input_split_sizes=recv_counts.tolist(), group=group)
    return out.cpu().numpy(), send_counts


class PartitionedCheby:
    """``cheby_op`` on one rank's row block of a partitioned Laplacian.

    ``step`` / ``gather_rows`` default to the CUDA kernels behind the C ABI; the CPU
    (gloo) tests of the host logic inject NumPy stand-ins.  There is no automatic
    fallback: without an injected backend a CUDA device is required.
    """

    def __init__(self, plan, dtype=None, device=None, group=None, backend=None, overlap=None,
                 exchange=None):
        import torch
        self.plan, self.group = plan, group
        # 'p2p': boundary rows are stored straight into the neighbours' halo rows over
        # NVLink peer memory, flags order the steps (csrc/halo.cu); 'nccl': pack +
        # all_to_all_single.  Default: p2p on GPUs, collective on the CPU test backend.
        self.exchange = exchange
        self.fuse_halo = True
        self._windows = {}
        self._seq = 0
        self.backend = backend if backend is not None else _CudaBackend(device)
        self.device = self.backend.device
        self.dtype = dtype if dtype is not None else torch.float32
        # Splitting a step into boundary + interior launches costs launches and tile
        # ramp-up; it pays only when the exchange itself is long (a sub-MB halo runs
        # faster unsplit).  None = decide per call from the halo size.
        self.overlap = overlap
        self.overlap_min_bytes = 16 << 20
        self.p2p_max_halo_fraction = 0.25
        t = lambda a, dt: (a if torch.is_tensor(a) else torch.from_numpy(
            np.ascontiguousarray(a))).to(device=self.device, dtype=dt)
        self.indptr = t(plan.indptr, torch.int32)
        self.indices = t(plan.indices, torch.int32)
        self.data = t(plan.data, self.dtype)
        self.perm = t(plan.perm, torch.int64)
        self.send_idx = t(plan.send_idx, torch.int64)
        self.in_splits = [int(v) for v in plan.send_counts]
        self.out_splits = [int(v) for v in plan.recv_counts]
        self._tile_plans = {}
        self._modes = {}
        self.bytes_sent_per_step = 0

    # ------------------------------------------------------------------ pieces
    def _exchange(self, buf, nsig):
        """Fill the halo rows of ``buf`` (n_local + n_halo, nsig) from the owners."""
        import torch.distributed as dist
        p = self.plan
        if p.parts == 1:
            return
        send = self.backend.gather_rows(buf, self.send_idx, nsig)
        self.bytes_sent_per_step = send.numel() * send.element_size()
        dist.all_to_all_single(buf[p.n_local:], send, output_split_sizes=self.out_splits,
                               input_split_sizes=self.in_splits, group=self.group)

    def _exchange_mode(self, nsig):
        """'p2p' or 'nccl' for this signal width -- the SAME answer on every rank.

        A rank-local choice deadlocks near the threshold (one rank enters the peer-window
        set-up, its neighbour the all-to-all), so the inputs of the decision are reduced over
        the group once per width: the largest halo of any rank decides the size rule, and
        p2p is used only if every rank reports that its neighbours are peer-reachable
        (same host, cudaDeviceCanAccessPeer); otherwise everybody falls back to NCCL.
        """
        import torch
        import torch.distributed as dist
        if nsig in self._modes:
            return self._modes[nsig]
        p = self.plan
        item = torch.empty((), dtype=self.dtype).element_size()
        halo_bytes = p.n_halo * nsig * item
        if not self.backend.has_streams or p.parts == 1:
            mode = self.exchange or "nccl"
        else:
            ok = 1 if self.backend.peers_reachable(self) else 0
            ratio_ppm = int(1e6 * p.n_halo / max(p.n_local, 1))
            t = torch.tensor([halo_bytes, -ok, ratio_ppm], dtype=torch.int64, device=self.device)
            dist.all_reduce(t, op=dist.ReduceOp.MAX, group=self.group)
            max_halo, all_ok, max_ratio = int(t[0].item()), int(t[1].item()) == -1, int(t[2].item())
            if self.exchange == "nccl" or not all_ok:
                mode = "nccl"
            elif self.exchange == "p2p":
                mode = "p2p"
            else:
                # peer stores from the step kernel's epilogue suit a halo that is a thin shell of
                # the block (k-NN / grid cuts: boundary rows are few and leave first); a halo as
                # large as the block itself (SBM: every row is a boundary row) moves better as
                # one packed transfer per peer
                thin = max_ratio <= int(1e6 * self.p2p_max_halo_fraction)
                mode = "p2p" if (thin or max_halo < self.overlap_min_bytes) else "nccl"
        self._modes[nsig] = mode
        return mode

    def _tile_plan(self, nsig, nscales):
        key = (nsig, nscales)
        if key not in self._tile_plans:
            self._tile_plans[key] = self.backend.tile_plan(self, nsig, nscales)
        return self._tile_plans[key]

    # ---------------------------------------------------------------- operator
    def cheby_op(self, lmax, c, x, local_order=False, clenshaw=None):
        """r = cheby_op(L, c, x) restricted to this rank's rows.

        x : (n_local, nsig) tensor on ``self.device`` (original local row order
            unless ``local_order``); returns (nscales, n_local, nsig) in the same order.
        clenshaw : single-filter calls on the peer-memory path default to Clenshaw's backward
            recurrence (one pass less over the block per order, same value, different
            rounding -- as on one GPU); ``False`` keeps the reference's operation order, which
            is bit-identical to the single-GPU forward recurrence.
        """
        import torch
        p = self.plan
        c = np.atleast_2d(np.asarray(c, dtype=np.float64))
        nscales, M = c.shape
        if M < 2:
            raise TypeError("The coefficients have an invalid shape")
        if x.shape[0] != p.n_local:
            raise ValueError("First dimension must be the number of local vertices")
        nsig = int(x.shape[1])
        n, nb = p.n_local, p.n_boundary
        ext = n + p.n_halo
        # Small halos (k-NN / grid cuts: < 1 MB): the exchange fused into the step kernel
        # wins.  Huge halos (SBM: hundreds of MB per step): one packed NCCL transfer
        # overlapped with the interior rows beats 128-byte peer stores.
        mode = self._exchange_mode(nsig)
        if mode == "p2p":
            return self._cheby_op_p2p(lmax, c, x, local_order,
                                      True if clenshaw is None else clenshaw)
        bufs = [torch.empty((ext, nsig), dtype=self.dtype, device=self.device) for _ in range(2)]
        xin = x.to(self.dtype)
        be = self.backend
        if local_order:
            bufs[0][:n] = xin
        elif be.has_streams:
            be.move_rows(xin.contiguous(), self.perm, bufs[0], scatter=False)
        else:
            bufs[0][:n] = xin.index_select(0, self.perm)
        r = torch.empty((nscales, n, nsig), dtype=self.dtype, device=self.device)
        plan = self._tile_plan(nsig, nscales)
        halo_bytes = p.n_halo * nsig * bufs[0].element_size()
        overlap = self.overlap if self.overlap is not None else halo_bytes >= self.overlap_min_bytes
        overlap = bool(overlap) and be.has_streams and p.parts > 1
        if overlap and p.send_idx.size and int(p.send_idx.max()) >= p.n_boundary:
            overlap = False          # non-symmetric pattern: sent rows are not all boundary rows
        self._exchange(bufs[0], nsig)                       # halo of T_0
        cur, old = 0, 1
        for k in range(1, M):
            first = k == 1
            ck = np.ascontiguousarray(c[:, k])
            c0 = np.ascontiguousarray(c[:, 0])
            coef = (2.0 / lmax, -1.0, 0.0) if first else (4.0 / lmax, -2.0, -1.0)
            # T_k overwrites T_{k-2} (row-local); for k == 1 it goes to the spare buffer
            x_cur, x_new = bufs[cur], bufs[old]
            args = (self, first, x_cur, x_new, x_new, r, nsig, nscales, ck, c0, coef, plan)
            last = k == M - 1
            if overlap and not last:
                be.step(*args, rows=(0, nb))
                be.fork_exchange(lambda: self._exchange(x_new, nsig))
                be.step(*args, rows=(nb, n))
                be.join_exchange()
            else:
                be.step(*args, rows=(0, n))
                if not last:
                    self._exchange(x_new, nsig)
            cur, old = old, cur
        if local_order:
            return r
        out = torch.empty_like(r)
        if be.has_streams:
            for i in range(nscales):
                be.move_rows(r[i], self.perm, out[i], scatter=True)
        else:
            out[:, self.perm] = r
        return out

    def filter_pinned(self, lmax, c, xh, clenshaw=None):
        """``cheby_op`` for a pinned HOST block (n_local, nsig) in the original row order: column
        chunks are uploaded / filtered / downloaded as a three-stream pipeline
        (filters/pipeline.py).  Returns a pinned host tensor (nscales, n_local, nsig)."""
        from .filters import pipeline
        c = np.atleast_2d(np.asarray(c, dtype=np.float64))
        p = self.plan          # the chunk width is derived from rank-independent sizes
        chunks = pipeline.chunk_plan(p.n_global // p.parts, int(xh.shape[1]), xh.element_size())
        return pipeline.run_pinned(lambda xc: self.cheby_op(lmax, c, xc, clenshaw=clenshaw),
                                   self.device, self.dtype, xh, c.shape[0], chunks=chunks)

    # ------------------------------------------------------------------- lmax
    def spmv(self, v):
        """(L v) restricted to this rank's rows; v: (n_local,) in local order."""
        import torch
        p = self.plan
        buf = torch.empty((p.n_local + p.n_halo, 1), dtype=self.dtype, device=self.device)
        buf[:p.n_local, 0] = v
        self._exchange(buf, 1)
        return self.backend.spmm(self, buf)[:, 0]

    def estimate_lmax(self, method="lanczos", seed=0, tol=5e-3, max_steps=400, polish_steps=60,
                      lap_type="combinatorial"):
        """Distributed ``Graph.estimate_lmax`` (graph.py:858-931) for the partitioned L.

        'lanczos': the same three-term recurrence and stopping rule as the single-GPU
        engine (``graphs.graph.ritz_check``); the operator is the local SpMM after a halo
        exchange, the two scalars per step are all-reduced.  Returns 1.01 * theta.
        'bounds': the minimum of the reference's four algebraic bounds (graph.py:933-960), the
        same value ``Graph.estimate_lmax('bounds')`` returns for the assembled graph.
        """
        import torch
        import torch.distributed as dist
        from .graphs.graph import ritz_check
        p = self.plan

        def allsum(t):
            if p.parts > 1:
                dist.all_reduce(t, group=self.group)
            return t
        if method == "bounds":
            return self._upper_bound(lap_type)
        if method != "lanczos":
            raise ValueError("Unknown method {}".format(method))
        gen = torch.Generator(device=self.device).manual_seed(seed * 7919 + p.rank)
        v = torch.rand(p.n_local, device=self.device, dtype=torch.float64, generator=gen) * 2 - 1
        v = (v / allsum((v * v).sum().reshape(1)).sqrt()).to(self.dtype)
        v_prev, beta_prev = None, 0.0
        alphas, betas = [], []
        cap = int(min(p.n_global, max_steps))
        theta, converged = 0.0, False
        for j in range(cap):
            w = self.spmv(v).double()
            alpha = float(allsum((w * v.double()).sum().reshape(1)).item())
            w = w - alpha * v.double()
            if v_prev is not None:
                w = w - beta_prev * v_prev.double()
            beta = float(allsum((w * w).sum().reshape(1)).sqrt().item())
            alphas.append(alpha)
            betas.append(beta)
            done = j + 1
            if done >= 10 and (done - 10) % 5 == 0 or done == cap or beta == 0.0:
                theta, _, stop, ref_rule = ritz_check(np.array(alphas), np.array(betas), tol,
                                                      self.dtype == torch.float32,
                                                      done >= polish_steps)
                converged = converged or ref_rule
                if stop:
                    return 1.01 * theta
            if beta == 0.0:
                break
            v_prev, beta_prev = v, beta
            v = (w / beta).to(self.dtype)
        if converged or cap == p.n_global:
            return 1.01 * theta
        raise ValueError("The Lanczos method did not converge. Try to use bounds.")

    def _upper_bound(self, lap_type="combinatorial"):
        """``Graph._get_upper_bound`` (graph.py:933-960) for the partitioned Laplacian: the minimum
        of N max W, 2 max dw, max over edges (dw_s + dw_t) and Merris' max(dw + (W dw) / dw) --
        2 for the normalized Laplacian.  W and dw are read off the rows of L = D - W (graphs
        without self-loops: L_ii = dw_i, L_ij = -w_ij); the weighted degrees of the halo columns
        come from one halo exchange, the maxima from all-reduces.  A NaN Merris bound (isolated
        vertex) is skipped like Python's ``min`` skips a trailing NaN in the reference."""
        import torch
        import torch.distributed as dist
        if lap_type == "normalized":
            return 2
        if lap_type != "combinatorial":
            raise ValueError("Unknown Laplacian type {}".format(lap_type))
        p = self.plan
        n = p.n_local
        dev = self.device
        row_of = row_ids(self.indptr)
        idx, val = self.indices.long(), self.data.double()
        on_diag = idx == row_of
        dw = torch.zeros(n, dtype=torch.float64, device=dev)
        dw.index_add_(0, row_of[on_diag], val[on_diag])
        ext = torch.zeros((n + p.n_halo, 1), dtype=self.dtype, device=dev)
        ext[:n, 0] = dw.to(self.dtype)
        self._exchange(ext, 1)                           # dw of the halo columns
        dw_ext = ext[:, 0].double()
        dw_ext[:n] = dw
        off = ~on_diag
        w, r_off, c_off = -val[off], row_of[off], idx[off]
        neg = torch.full((1,), -float("inf"), dtype=torch.float64, device=dev)
        has_edges = w.numel() > 0
        wd = torch.zeros(n, dtype=torch.float64, device=dev)
        if has_edges:
            wd.index_add_(0, r_off, w * dw_ext[c_off])
        isolated = bool((dw == 0).any().item()) if n else False
        merris = (dw + wd / dw).max().reshape(1) if (n and not isolated) else neg.clone()
        tops = torch.cat([w.max().reshape(1) if has_edges else neg.clone(),
                          dw.max().reshape(1) if n else neg.clone(),
                          (dw[r_off] + dw_ext[c_off]).max().reshape(1) if has_edges else neg.clone(),
                          merris,
                          torch.tensor([1.0 if isolated else 0.0], dtype=torch.float64, device=dev)])
        if p.parts > 1:
            dist.all_reduce(tops, op=dist.ReduceOp.MAX, group=self.group)
        w_max, dw_max, edge_max, merris_max, any_isolated = (float(v) for v in tops.tolist())
        bounds = [p.n_global * w_max if w_max > -float("inf") else 0.0, 2 * dw_max]
        if edge_max > -float("inf"):
            bounds.append(edge_max)
        if not any_isolated:
            bounds.append(merris_max)
        return float(min(bounds))

    def _cheby_op_p2p(self, lmax, c, x, local_order, clenshaw=False):
        """The whole call is ONE C entry point, ``gsp_cheby_op_dist_*`` (csrc/dist.cu): entry
        barrier, halo of T_0, K steps with the exchange fused into the step kernel (float32 +
        tile plan; wait / step / push kernels otherwise).  Python only owns the plan."""
        import ctypes
        import torch
        p = self.plan
        c = np.ascontiguousarray(np.atleast_2d(np.asarray(c, dtype=np.float64)))
        nscales, M = c.shape
        nsig = int(x.shape[1])
        n = p.n_local
        if nsig not in self._windows:
            self._windows[nsig] = PeerWindow(self, nsig)
        win = self._windows[nsig]
        xin = x.to(self.dtype).contiguous()
        use_clenshaw = bool(clenshaw) and nscales == 1 and M >= 3
        r = torch.empty((nscales, n, nsig), dtype=self.dtype, device=self.device)
        plan = self._tile_plan(nsig, nscales)
        win.dist_plan.separate_exchange = 0 if self.fuse_halo else 1
        seq = ctypes.c_uint64(self._seq)
        # the row permutation (boundary rows first) is applied inside the call: the input is
        # gathered straight into the window, the result is stored to the caller's rows
        win.dist_plan.perm = None if local_order else self.perm.data_ptr()
        with torch.cuda.device(self.device):
            nat.call("gsp_cheby_op_dist_" + nat.suffix(self.dtype), win.dist_plan, plan,
                     nat.f64(lmax), c, nat.i32(nscales), nat.i32(M), xin, nat.i64(nsig), r,
                     nat.i32(1 if use_clenshaw else 0), ctypes.byref(seq),
                     nat.stream_ptr(self.device))
        self._seq = int(seq.value)
        self.bytes_sent_per_step = int(win.src_row.numel()) * nsig * xin.element_size()
        return r


def _neighbors(plan):
    """The ranks this rank exchanges halo rows with, ascending."""
    return [q for q in range(plan.parts)
            if q != plan.rank and (plan.send_counts[q] > 0 or plan.recv_counts[q] > 0)]


class PeerTables:
    """The device tables of one rank's ``gsp_dist_plan`` and the plan itself (``dist_plan``).

    Pure host computation from the rank's ``HaloPlan`` and what every rank publishes about its
    window: ``infos[q] = (n_local, recv_counts, buf_bytes)`` of rank q, and ``bases[q]``, the
    device address at which THIS rank sees rank q's window (its own for q == rank; None for
    ranks that are not neighbours).  A window is ``buf0 | buf1 | buf2 | flags[P] (uint64) |
    push counter (uint32) | fused counter (uint64, at +8)``.  ``indptr`` / ``indices`` /
    ``data`` / ``send_idx`` are the rank's device tensors.  The tables live as long as this
    object; ``dist_plan`` points into them.
    """

    def __init__(self, plan, infos, bases, indptr, indices, data, send_idx, n_bufs=3):
        import torch
        p = plan
        dev = send_idx.device
        self.neighbors = _neighbors(p)
        # destination row of every packed row: the slot the neighbour reserved for it
        dst_peer, dst_row = [], []
        for q in range(p.parts):
            cnt = int(p.send_counts[q])
            if cnt == 0:
                continue
            n_local_q, recv_q = infos[q][0], infos[q][1]
            first = n_local_q + int(sum(recv_q[:p.rank]))     # q's halo slots are owner-ordered
            dst_peer.append(np.full(cnt, q, dtype=np.int32))
            dst_row.append(first + np.arange(cnt, dtype=np.int64))
        cat = lambda parts, dt: torch.from_numpy(
            np.concatenate(parts) if parts else np.zeros(0, dtype=dt)).to(dev)
        self.dst_peer = cat(dst_peer, np.int32)
        self.dst_row = cat(dst_row, np.int64)
        self.src_row = send_idx
        base_tab = np.zeros((n_bufs, p.parts), dtype=np.int64)
        for q in self.neighbors:
            for b in range(n_bufs):
                base_tab[b, q] = bases[q] + b * infos[q][2]
        self.peer_base = torch.from_numpy(base_tab).to(dev)                  # pointers as int64
        flag_tab = np.array([bases[q] + n_bufs * infos[q][2] + 8 * p.rank
                             for q in self.neighbors], dtype=np.int64)
        self.peer_flags = torch.from_numpy(flag_tab).to(dev)
        self.neighbor_ids = torch.from_numpy(np.asarray(self.neighbors, dtype=np.int32)).to(dev)
        # the same send list as a CSR over the local rows, for the fused epilogue push
        src = p.send_idx
        order = np.argsort(src, kind="stable")
        self.n_push_rows = int(src.max()) + 1 if src.size else 0
        ptr = np.zeros(self.n_push_rows + 1, dtype=np.int64)
        np.add.at(ptr, src + 1, 1)
        self.push_ptr = torch.from_numpy(np.cumsum(ptr).astype(np.int32)).to(dev)
        self.push_peer = self.dst_peer[torch.from_numpy(order).to(dev)].contiguous()
        self.push_row = self.dst_row[torch.from_numpy(order).to(dev)].contiguous()
        own, buf_bytes = bases[p.rank], infos[p.rank][2]
        flags_ptr = own + n_bufs * buf_bytes
        counter_ptr = flags_ptr + 8 * p.parts
        d = nat.DistPlan()
        d.n_local, d.n_halo, d.nnz = p.n_local, p.n_halo, p.nnz
        d.indptr, d.indices, d.data = indptr.data_ptr(), indices.data_ptr(), data.data_ptr()
        for b in range(n_bufs):
            d.buf[b] = own + b * buf_bytes
            d.peer_base[b] = self.peer_base[b].data_ptr()
        d.peer_flags = self.peer_flags.data_ptr()
        d.flags = flags_ptr
        d.neighbor_ids = self.neighbor_ids.data_ptr()
        d.n_neighbors = len(self.neighbors)
        d.push_counter, d.fused_counter = counter_ptr, counter_ptr + 8
        d.n_send = int(self.src_row.numel())
        d.src_row, d.dst_peer, d.dst_row = (self.src_row.data_ptr(), self.dst_peer.data_ptr(),
                                            self.dst_row.data_ptr())
        d.n_push_rows = self.n_push_rows
        d.push_ptr, d.push_peer, d.push_row = (self.push_ptr.data_ptr(), self.push_peer.data_ptr(),
                                               self.push_row.data_ptr())
        d.n_boundary_rows = p.n_true_boundary
        self.dist_plan = d


class PeerWindow:
    """State buffers + flags of one rank for one signal width, IPC-mapped by its neighbours.

    One cudaMalloc'ed block: buf0 | buf1 | buf2 | flags[P] (uint64) | push counters.  ``push``
    stores this rank's boundary rows into the neighbours' halo rows and publishes a
    sequence number; ``wait`` stalls the stream until the neighbours published it (both live
    in the library: csrc/halo.cu, csrc/dist.cu -- this class only owns the memory and the tables).
    """

    def __init__(self, op, nsig):
        import ctypes
        import torch
        import torch.distributed as dist
        p, self.op, self.nsig = op.plan, op, nsig
        item = torch.empty((), dtype=op.dtype).element_size()
        ext = p.n_local + p.n_halo
        self.buf_bytes = ((ext * nsig * item + 255) // 256) * 256
        self.n_bufs = 3                       # the Clenshaw form keeps x, b_{k+1} and b_{k+2}
        flag_off = self.n_bufs * self.buf_bytes
        total = flag_off + 8 * p.parts + 256
        ptr = ctypes.c_void_p()
        handle = (ctypes.c_ubyte * 64)()
        with torch.cuda.device(op.device):
            nat.call("gsp_ipc_alloc", ctypes.c_size_t(total), ctypes.byref(ptr), handle)
        self.base = int(ptr.value)
        self.bufs = [_wrap(self.base + b * self.buf_bytes, (ext, nsig), op.dtype, op.device)
                     for b in range(self.n_bufs)]
        # everybody learns everybody's handle, block size and halo layout
        info = [None] * p.parts
        dist.all_gather_object(info, (bytes(handle), int(p.n_local), p.recv_counts.tolist(),
                                      int(self.buf_bytes)), group=op.group)
        self.opened = {}
        for q in _neighbors(p):
            qptr = ctypes.c_void_p()
            hq = (ctypes.c_ubyte * 64).from_buffer_copy(info[q][0])
            with torch.cuda.device(op.device):
                nat.call("gsp_ipc_open", hq, ctypes.byref(qptr))
            self.opened[q] = int(qptr.value)
        bases = [self.base if q == p.rank else self.opened.get(q) for q in range(p.parts)]
        self.tables = PeerTables(p, [i[1:] for i in info], bases, op.indptr, op.indices, op.data,
                                 op.send_idx, self.n_bufs)
        self.src_row = op.send_idx
        self.dist_plan = self.tables.dist_plan
        torch.cuda.synchronize(op.device)
        if p.parts > 1:
            dist.barrier(group=op.group)

    def close(self):
        import ctypes
        torch = nat.require_cuda()
        torch.cuda.synchronize(self.op.device)
        for qptr in self.opened.values():
            nat.call("gsp_ipc_close", ctypes.c_void_p(qptr))
        self.opened = {}
        if self.base:
            nat.call("gsp_ipc_free", ctypes.c_void_p(self.base))
            self.base = 0


class _RawCuda:
    def __init__(self, ptr, shape, typestr):
        self.__cuda_array_interface__ = {"data": (ptr, False), "shape": tuple(shape),
                                         "typestr": typestr, "version": 3, "strides": None}


def _wrap(ptr, shape, dtype, device):
    """A torch view (no copy, no ownership) of raw device memory."""
    torch = nat.require_cuda()
    typestr = {torch.float32: "<f4", torch.float64: "<f8"}[dtype]
    with torch.cuda.device(device):
        return torch.as_tensor(_RawCuda(ptr, shape, typestr), device=device)


class _CudaBackend:
    has_streams = True

    def __init__(self, device=None):
        torch = nat.require_cuda()
        self.device = torch.device(device if device is not None
                                   else "cuda:%d" % torch.cuda.current_device())
        self.comm_stream = torch.cuda.Stream(device=self.device)
        self._evt = None

    def peers_reachable(self, op):
        """True if every neighbour of this rank is on this host and peer-mappable."""
        import socket
        import torch.distributed as dist
        torch = nat.require_cuda()
        p = op.plan
        info = [None] * p.parts
        dist.all_gather_object(info, (socket.gethostname(), self.device.index), group=op.group)
        me = info[p.rank]
        for q in range(p.parts):
            if q == p.rank or not (p.send_counts[q] > 0 or p.recv_counts[q] > 0):
                continue
            host, dev = info[q]
            if host != me[0]:
                return False
            if dev != me[1] and not torch.cuda.can_device_access_peer(me[1], dev):
                return False
        return True

    def tile_plan(self, op, nsig, nscales):
        torch = nat.require_cuda()
        if op.dtype != torch.float32:
            return None
        plan = nat.TilePlan()
        with torch.cuda.device(self.device):
            nat.call("gsp_cheby_tile_plan", nat.i64(op.plan.n_local), op.indptr, nat.i64(nsig),
                     nat.i32(nscales), plan, nat.stream_ptr(self.device))
        return plan if plan.rows_per_tile > 0 else None

    def gather_rows(self, buf, idx, nsig):
        torch = nat.require_cuda()
        out = torch.empty((idx.numel(), nsig), dtype=buf.dtype, device=self.device)
        with torch.cuda.device(self.device):
            nat.call("gsp_gather_rows_" + nat.suffix(buf.dtype), nat.i64(idx.numel()), idx, buf,
                     nat.i64(nsig), out, nat.stream_ptr(self.device))
        return out

    def move_rows(self, src, idx, dst, scatter):
        """dst[i,:] = src[idx[i],:] (scatter: dst[idx[i],:] = src[i,:]) for the rows of idx."""
        torch = nat.require_cuda()
        with torch.cuda.device(self.device):
            nat.call(("gsp_scatter_rows_" if scatter else "gsp_gather_rows_") + nat.suffix(src.dtype),
                     nat.i64(idx.numel()), idx, src, nat.i64(src.shape[1]), dst,
                     nat.stream_ptr(self.device))

    def step(self, op, first, x_cur, x_old, x_new, r, nsig, nscales, ck, c0, coef, plan, rows):
        torch = nat.require_cuda()
        if rows[1] <= rows[0]:
            return
        with torch.cuda.device(self.device):
            nat.call("gsp_cheby_step_" + nat.suffix(op.dtype), nat.i32(1 if first else 0),
                     nat.i64(rows[0]), nat.i64(rows[1]), nat.i64(op.plan.nnz), op.indptr,
                     op.indices, op.data, x_cur, None if first else x_old, x_new, r,
                     nat.i64(op.plan.n_local), nat.i64(nsig), nat.i32(nscales), ck, c0,
                     nat.f64(coef[0]), nat.f64(coef[1]), nat.f64(coef[2]), plan,
                     nat.stream_ptr(self.device))

    def spmm(self, op, x_ext):
        """y = L_local x_ext: (n_local, width) from the extended (n_local + n_halo, width)."""
        torch = nat.require_cuda()
        width = int(x_ext.shape[1])
        y = torch.empty((op.plan.n_local, width), dtype=op.dtype, device=self.device)
        with torch.cuda.device(self.device):
            nat.call("gsp_spmm_" + nat.suffix(op.dtype), nat.i64(op.plan.n_local), op.indptr,
                     op.indices, op.data, x_ext, nat.i64(width), y, nat.stream_ptr(self.device))
        return y

    def fork_exchange(self, fn):
        """Run the pack + all-to-all on the side stream, after what is queued so far."""
        torch = nat.require_cuda()
        main = torch.cuda.current_stream(self.device)
        self.comm_stream.wait_stream(main)
        with torch.cuda.stream(self.comm_stream):
            fn()
            self._evt = self.comm_stream.record_event()

    def join_exchange(self):
        torch = nat.require_cuda()
        if self._evt is not None:
            torch.cuda.current_stream(self.device).wait_event(self._evt)
            self._evt = None
