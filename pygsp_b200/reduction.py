"""Callers of the Chebyshev filtering path in ``pygsp/reduction.py`` (SURVEY.md 8f rank 3).

``interpolate`` (reduction.py:150-193), ``pyramid_analysis`` (:384-449) and the direct branch
of ``pyramid_synthesis`` (:504-514): every step of the Kron pyramid is a Chebyshev filter --
the analysis filter ``h`` and the order-100 Green kernel ``1 / (eps + x)`` of the
interpolation -- and runs on the CUDA engine through :class:`pygsp_b200.filters.Filter`.
The multiresolution sequence itself runs on the device too (DESIGN.md section 4.11):
``graph_multiresolution`` (largest-eigenvector down-sampling by Chebyshev-filtered subspace
iteration), :func:`kron_reduction` (independent Schur blocks per component of the removed
vertices, csrc/schur.cu, or random-walk samples of the Schur complement that never form a dense
block, csrc/schur_walk.cu and DESIGN.md section 4.23) and :func:`graph_sparsify` (effective resistances from one float64
factor or, past its size, from a Johnson-Lindenstrauss sketch solved by block CG, csrc/resistance.cu
and DESIGN.md section 4.22; seeded Philox sampling).  :func:`tree_multiresolution` (reduction.py:633-787, which
cannot run in the reference) coarsens a tree to its even-depth vertices level after level: the
tree is rooted by an Euler tour ranked by pointer jumping, in O(log N) launches whatever its depth,
and each level is a few O(N) kernels (csrc/tree.cu, DESIGN.md section 4.21).

A graph of the sequence carries ``G.mr = {'idx': kept vertices of the level above,
'K_reg': ...}`` like the reference's.  Shapes: the reference keeps consistent shapes only for
column-vector signals (a 1-D signal is broadcast to (N, N) at reduction.py:447); here a signal is
(N,) or (N, Nv), every coefficient block is returned 2-D (n_level, Nv), and Nv columns mean Nv
independent signals.  The least-squares synthesis (reduction.py:534-630) is broken in the
reference (NameError at :593) and has no oracle; ``least_squares=True`` raises.
"""
import numpy as np
from scipy import sparse

from . import _native as nat
from . import filters
from . import utils
from .graphs.csr import DeviceCSR, row_ids

logger = utils.build_logger(__name__)


# Components of the removed vertices with at most SMALL_MAX vertices whose blocks fit in
# _SMALL_SMEM bytes of shared memory are reduced by the one-CTA kernel (gsp_schur_small_f64);
# the others by a dense float64 Cholesky (cuSOLVER).  Chosen with tools/multiresolution_probe.py
# (DESIGN.md section 4.11).
SMALL_MAX = 64
_SMALL_SMEM = 96 * 1024


def _ctx():
    torch = nat.require_cuda()
    return torch, torch.device("cuda:%d" % torch.cuda.current_device())


def _device_matrix(L, device):
    """A host (SciPy / NumPy) or device square matrix as a canonical float64 DeviceCSR without
    stored zeros: an explicit zero is not an edge (it must not join two components)."""
    torch = nat.require_cuda()
    if isinstance(L, DeviceCSR):
        M = DeviceCSR(L.indptr, L.indices, L.data.to(torch.float64), L.shape)
        return M.eliminate_zeros() if bool((M.data == 0).any()) else M
    if hasattr(L, "to_scipy"):
        L = L.to_scipy()
    host = sparse.csr_matrix(L, dtype=np.float64)
    if host.shape[0] != host.shape[1]:
        raise ValueError("The matrix must be square.")
    host.sum_duplicates()
    host.eliminate_zeros()
    host.sort_indices()
    return DeviceCSR.from_scipy(host, torch.float64, device)


def _call(name, *args):
    nat.call(name, *args, nat.stream_ptr())


def _split(M, ind):
    """(slot, rem, R, r_rows) of the kept vertices ``ind`` (host int64, distinct) of the float64
    DeviceCSR M: slot[v] = -1 - (index of v in ind) for a kept vertex, 0 for a removed one (int32);
    rem the removed vertices, ascending (int32); R, r_rows = M.induced(ind), unsorted triplets of
    M[ind][:, ind]."""
    torch = nat.require_cuda()
    dev, n, m = M.device, M.shape[0], len(ind)
    keep = torch.from_numpy(np.ascontiguousarray(ind, dtype=np.int32)).to(dev)
    slot = torch.zeros(n, dtype=torch.int32, device=dev)
    slot[keep.long()] = -1 - torch.arange(m, dtype=torch.int32, device=dev)
    rem = torch.nonzero(slot == 0).flatten().to(torch.int32)
    R, r_rows = M.induced(keep)
    return slot, rem, R, r_rows


def _removed_components(M, slot, rem, m):
    """Connected components of the removed vertices ``rem`` (non-empty) of M and the kept
    neighbours of each: (nc, cvert, cptr, sizes, comp_of, bidx, nbs, bptr).  cvert lists the
    removed vertices component by component, component c at cvert[cptr[c] .. cptr[c + 1]) (int32);
    sizes its sizes and comp_of[v] the component of v, -1 for a kept vertex (int64); its kept
    neighbours, in increasing kept index, at bidx[bptr[c] .. bptr[c + 1]) (int32, bptr int64),
    nbs = their numbers.  slot[v] of a removed vertex becomes its position in its component."""
    torch = nat.require_cuda()
    dev, n, nr = M.device, M.shape[0], int(rem.numel())
    S, _ = M.induced(rem, increasing=True)
    labels = torch.empty(nr, dtype=torch.int32, device=dev)
    _call("gsp_cc_labels_f64", nat.i64(nr), S.indptr, S.indices, S.data, nat.i32(0), labels, None)
    perm = torch.empty(nr, dtype=torch.int32, device=dev)
    cptr = torch.empty(nr + 1, dtype=torch.int32, device=dev)
    ncomp = torch.empty(1, dtype=torch.int64, device=dev)
    _call("gsp_component_order", nat.i64(nr), labels, perm, cptr, ncomp)
    nc = int(ncomp.item())
    cptr = cptr[:nc + 1].contiguous()
    cvert = rem[perm.long()].contiguous()
    sizes = (cptr[1:] - cptr[:-1]).long()
    comp_of_pos = torch.repeat_interleave(torch.arange(nc, device=dev), sizes)
    slot[cvert.long()] = (torch.arange(nr, device=dev) - cptr[comp_of_pos].long()).to(torch.int32)
    comp_of = torch.full((n,), -1, dtype=torch.int64, device=dev)
    comp_of[cvert.long()] = comp_of_pos

    # kept neighbours of every component, in increasing kept index
    rows, cols = row_ids(M.indptr), M.indices.long()
    edge = (comp_of[rows] >= 0) & (slot[cols] < 0)
    keys = torch.unique(comp_of[rows[edge]] * m + (-1 - slot[cols[edge]].long()))
    bcomp, bidx = keys // m, (keys % m).to(torch.int32).contiguous()
    nbs = torch.bincount(bcomp, minlength=nc)
    bptr = torch.zeros(nc + 1, dtype=torch.int64, device=dev)
    bptr[1:] = torch.cumsum(nbs, 0)
    return nc, cvert, cptr, sizes, comp_of, bidx, nbs, bptr


def _schur(M, ind, small_max=None):
    """Kron reduction of the symmetric float64 DeviceCSR M onto the vertices ``ind`` (host int64
    array, distinct), as a canonical float64 DeviceCSR in the order of ``ind``.

    M_red - sum_S M_BS M_SS^-1 M_SB over the connected components S of the removed vertices
    (B: S's kept neighbours): every component is an independent block (csrc/schur.cu).
    ``small_max`` overrides SMALL_MAX (tests compare the two paths on the same components).
    """
    torch = nat.require_cuda()
    dev, m = M.device, len(ind)
    small_max = SMALL_MAX if small_max is None else int(small_max)
    slot, rem, R, r_rows = _split(M, ind)
    nr = int(rem.numel())
    if nr == 0:
        return DeviceCSR.from_coo(r_rows, R.indices, R.data, (m, m))
    nc, cvert, cptr, sizes, _, bidx, nbs, bptr = _removed_components(M, slot, rem, m)
    out_len = nbs * nbs
    out_off = torch.zeros(nc + 1, dtype=torch.int64, device=dev)
    out_off[1:] = torch.cumsum(out_len, 0)
    total = int(out_off[-1].item())
    nnz_red = R.nnz
    if total + nnz_red >= 2 ** 31:
        raise ValueError("The Kron reduction would have {} entries before summation; at most "
                         "2^31 - 1 are supported.".format(total + nnz_red))

    # small components: one CTA each; the others: dense Cholesky.  A component without kept
    # neighbours contributes nothing (its M_SS may be singular) and is skipped.
    smem = 8 * (sizes * sizes + sizes + sizes * nbs) + 4 * nbs
    small = (sizes <= small_max) & (smem <= _SMALL_SMEM) & (nbs > 0)
    dense = (~small) & (nbs > 0)
    rows_out = torch.empty(total + nnz_red, dtype=torch.int32, device=dev)
    cols_out = torch.empty(total + nnz_red, dtype=torch.int32, device=dev)
    vals_out = torch.empty(total + nnz_red, dtype=torch.float64, device=dev)
    rows_out[total:], cols_out[total:], vals_out[total:] = r_rows, R.indices, R.data
    status = torch.zeros(1, dtype=torch.int32, device=dev)
    bptr32 = bptr.to(torch.int32).contiguous()
    comps = torch.nonzero(small).flatten().to(torch.int32).contiguous()
    if comps.numel():
        _call("gsp_schur_small_f64", M.indptr, M.indices, M.data, slot, cvert, cptr, bptr32, bidx,
              nat.i64(comps.numel()), comps, nat.i32(int(smem[small].max().item())),
              out_off, rows_out, cols_out, vals_out, status)
    dense_ids = torch.nonzero(dense).flatten().cpu().numpy()
    if dense_ids.size:
        host_c, host_b, host_o = (cptr.cpu().numpy(), bptr.cpu().numpy(),
                                  out_off.cpu().numpy())
        for c in dense_ids:
            c0, s = int(host_c[c]), int(host_c[c + 1] - host_c[c])
            b0, b = int(host_b[c]), int(host_b[c + 1] - host_b[c])
            A = torch.empty((s, s), dtype=torch.float64, device=dev)
            B = torch.empty((s, b), dtype=torch.float64, device=dev)
            bc = bidx[b0:b0 + b]
            _call("gsp_schur_gather_f64", M.indptr, M.indices, M.data, slot, cvert[c0:c0 + s],
                  nat.i64(s), bc, nat.i64(b), A, B)
            C, info = torch.linalg.cholesky_ex(A)
            if int(info.item()) != 0:
                status.fill_(1)
                continue
            Y = torch.linalg.solve_triangular(C, B, upper=False)
            del A, B, C
            K = Y.T @ Y
            o = int(host_o[c])
            vals_out[o:o + b * b] = (-0.5 * (K + K.T)).flatten()
            rows_out[o:o + b * b] = bc.repeat_interleave(b)
            cols_out[o:o + b * b] = bc.repeat(b)
    if int(status.item()):
        raise ValueError("Kron reduction: a block of the removed vertices is not positive "
                         "definite (the matrix is not a connected Laplacian-like matrix).")
    # components without kept neighbours emitted nothing: their slots are empty (b = 0)
    out = DeviceCSR.from_coo(rows_out, cols_out, vals_out, (m, m))
    # Every block is symmetric and M_red is, but the summation of duplicates need not associate
    # (i, j) and (j, i) alike; average with the transpose if any entry differs (the reference
    # symmetrises an almost symmetric result too, reduction.py:361-362).
    if _asymmetry(out):
        out = out.symmetrize("average")
    return out


def _asymmetry(M):
    """Number of stored entries of the float64 DeviceCSR M that differ from their transpose."""
    torch = nat.require_cuda()
    count = torch.zeros(1, dtype=torch.int64, device=M.device)
    _call("gsp_csr_asymmetry_f64", nat.i64(M.shape[0]), M.indptr, M.indices, M.data, count)
    return int(count.item())


def _check_symmetric(M, what="Kron reduction"):
    if _asymmetry(M):
        raise ValueError("{} on the device needs a symmetric matrix.".format(what))


# Kron reduction by random walks (csrc/schur_walk.cu, DESIGN.md section 4.23): bits of its status
_WALK_NEGATIVE, _WALK_NOT_DOMINANT, _WALK_CAPPED = 1, 2, 4
_KRON_METHODS = ("exact", "walks")
_WALK_MAX_STEPS = 2 ** 20


def _check_kron_method(method, samples, max_steps=1):
    if method not in _KRON_METHODS:
        raise ValueError("method must be 'exact' or 'walks', not {!r}.".format(method))
    if int(samples) < 1:
        raise ValueError("samples must be at least 1, not {}.".format(samples))
    if int(max_steps) < 1:
        raise ValueError("max_steps must be at least 1, not {}.".format(max_steps))


def _schur_walks(M, ind, samples, key, max_steps, excess=None, stats=None):
    """Kron reduction of the symmetric float64 DeviceCSR M onto the vertices ``ind`` (host int64
    array, distinct) by random-walk samples of the Schur complement, as a canonical float64
    DeviceCSR in the order of ``ind`` (csrc/schur_walk.cu).

    M is read as weights w_uv = -M_uv and an excess per vertex, an edge to a ground vertex:
    ``excess`` (a float64 device tensor, one value per vertex) or, when None, M_uu - sum_v w_uv,
    which must not fall below -1e-12 M_uu.  Every kept-kept edge and the excess of every kept vertex
    are exact samples; every other edge and the excess of every removed vertex are sampled
    ``samples`` times with the Philox key ``key``.  Components of the removed vertices without a
    kept neighbour contribute nothing and are not walked.  With nothing removed the result is
    M[ind][:, ind].  ``stats`` (a dict) receives the number of steps of every item ('steps').
    """
    torch = nat.require_cuda()
    dev, n, m = M.device, M.shape[0], len(ind)
    prefix = torch.empty(M.nnz, dtype=torch.float64, device=dev)
    total = torch.empty(n, dtype=torch.float64, device=dev)
    ex = torch.empty(n, dtype=torch.float64, device=dev)
    status = torch.zeros(1, dtype=torch.int32, device=dev)
    _call("gsp_walk_prep_f64", nat.i64(n), M.indptr, M.indices, M.data, excess, prefix, total, ex,
          status)
    flags = int(status.item())
    if flags & _WALK_NEGATIVE:
        raise ValueError("Kron reduction by random walks needs non-negative weights (the matrix "
                         "has a positive off-diagonal entry).")
    if flags & _WALK_NOT_DOMINANT:
        raise ValueError("Kron reduction by random walks needs a diagonally dominant matrix "
                         "(some M_uu - sum_v |M_uv| is below -1e-12 M_uu).")
    slot, rem, R, r_rows = _split(M, ind)
    if rem.numel() == 0:
        return DeviceCSR.from_coo(r_rows, R.indices, R.data, (m, m))
    _, _, _, _, comp_of, _, nbs, _ = _removed_components(M, slot, rem, m)
    dead = (comp_of >= 0) & (nbs[comp_of.clamp(min=0)] == 0)

    # items: the sampled edges (lower triangle, CSR order) and the ground edges of removed vertices
    rows, cols = row_ids(M.indptr), M.indices.long()
    removed = slot >= 0
    sampled = (rows > cols) & (removed[rows] | removed[cols]) & ~dead[rows]
    eu, ev = rows[sampled].to(torch.int32), cols[sampled].to(torch.int32)
    ew = (-M.data[sampled]).contiguous()
    gu = torch.nonzero(removed & ~dead & (ex > 0)).flatten().to(torch.int32)
    ne, ng = int(eu.numel()), int(gu.numel())

    # exact samples: every kept-kept edge as its Laplacian triplets, and the kept excesses
    kr, kc = r_rows.long(), R.indices.long()
    off = kr != kc
    kex = ex[torch.from_numpy(np.ascontiguousarray(ind, dtype=np.int64)).to(dev)]
    kx = torch.nonzero(kex > 0).flatten()
    x_rows = torch.cat([kr[off], kr[off], kx]).to(torch.int32)
    x_cols = torch.cat([kc[off], kr[off], kx]).to(torch.int32)
    x_vals = torch.cat([R.data[off], -R.data[off], kex[kx]])
    slots = (4 * ne + ng) * samples
    if (ne + ng) * samples >= 2 ** 31 or slots + int(x_rows.numel()) >= 2 ** 31:
        raise ValueError("The sampled Kron reduction would have {} items and {} entries before "
                         "summation; at most 2^31 - 1 are supported.".format(
                             (ne + ng) * samples, slots + int(x_rows.numel())))
    rows_out = torch.empty(slots, dtype=torch.int32, device=dev)
    cols_out = torch.empty(slots, dtype=torch.int32, device=dev)
    vals_out = torch.empty(slots, dtype=torch.float64, device=dev)
    steps = (torch.empty((ne + ng) * samples, dtype=torch.int32, device=dev)
             if stats is not None else None)
    _call("gsp_schur_walk_f64", M.indptr, M.indices, M.data, prefix, total, ex, slot, nat.i64(ne),
          eu, ev, ew, nat.i64(ng), gu, nat.i64(samples), nat.u64(key), nat.i64(max_steps),
          rows_out, cols_out, vals_out, steps, status)
    if int(status.item()) & _WALK_CAPPED:
        raise ValueError("Kron reduction by random walks: a walk took max_steps = {} steps "
                         "without reaching a kept vertex; raise max_steps or use "
                         "method='exact'.".format(max_steps))
    if stats is not None:
        stats["steps"] = steps
    hit = rows_out >= 0
    # one sort sums every entry's samples in emission order: (i, j) and (j, i) receive the same
    # values in the same order, so the result is exactly symmetric
    return DeviceCSR.from_coo(torch.cat([x_rows, rows_out[hit]]), torch.cat([x_cols, cols_out[hit]]),
                              torch.cat([x_vals, vals_out[hit]]), (m, m))


def _kept_ids(ind, n):
    ind = np.asarray(ind)
    if ind.dtype == bool:
        ind = np.flatnonzero(ind)
    ind = ind.astype(np.int64).reshape(-1)
    if ind.size and (ind.min() < 0 or ind.max() >= n or np.unique(ind).size != ind.size):
        raise ValueError("ind must list distinct vertices in [0, {}).".format(n))
    return ind


def _kron_graph(G, ind, method, samples, key, max_steps):
    """kron_reduction of a Graph onto the kept vertices ``ind``, with the walk key ``key``."""
    from .graphs import Graph
    torch = nat.require_cuda()
    if G.lap_type != "combinatorial":
        raise NotImplementedError("Unknown reduction for {} Laplacian.".format(G.lap_type))
    if G.is_directed():
        raise NotImplementedError("This method only work for undirected graphs.")
    ind = _kept_ids(ind, G.N)
    with torch.cuda.device(G.device):
        M = _device_matrix(G.L, G.device)
        if method == "walks":
            # the weights are -offdiag(L) and the excess exactly 0: a float32 graph's stored
            # diagonal is not exactly W 1
            L = _schur_walks(M, ind, samples, key, max_steps,
                             excess=torch.zeros(G.N, dtype=torch.float64, device=G.device))
        else:
            L = _schur(M, ind)
        rows = row_ids(L.indptr)
        off = rows != L.indices.long()
        return Graph.from_coo(rows[off], L.indices[off], -L.data[off], len(ind),
                              lap_type=G.lap_type, dtype=G.dtype, device=G.device,
                              coords=G.coords[ind] if hasattr(G, "coords") else None,
                              plotting=G.plotting)


def kron_reduction(G, ind, *, method="exact", samples=16, seed=None, max_steps=_WALK_MAX_STEPS):
    r"""Compute the Kron reduction (reduction.py:309-382).

    ``G``: a :class:`Graph` with a combinatorial Laplacian, or a symmetric sparse matrix
    (Laplacian-like, such as ``L + eps I``; SciPy, NumPy or a ``DeviceCSR``).  Unlike the
    reference, a non-symmetric matrix raises ``ValueError`` (each block is factored by Cholesky),
    and so does a matrix whose removed blocks are not positive definite.  ``ind``: the
    vertices to keep, in the order of the result.  The Schur complement
    ``L[ind, ind] - L[ind, comp] L[comp, comp]^-1 L[comp, ind]`` is computed on the device in
    float64, one independent block per connected component of the removed vertices
    (csrc/schur.cu).  A matrix in gives a SciPy CSR float64 matrix out; a graph in gives a graph
    on ``W = -offdiag(L_new)`` with the sliced coordinates, in the graph's dtype (weights that
    underflow in float32 are dropped).  The diagonal of ``L_new`` is dropped, as the reference's
    comment intends; its ``Snew`` correction (reduction.py:366-372) is not reproduced (DESIGN.md
    section 2).

    ``method`` (keyword-only, an addition the reference does not have): ``'exact'`` (the default)
    as above, or ``'walks'``, which never forms a dense block and so reaches graphs whose removed
    components are too large for one (DESIGN.md section 4.23).  It samples the Schur complement
    by random walks (Durfee, Kyng, Peebles, Rao and Sachdeva): every edge with a removed end, and
    the excess ``M_uu - sum_v |M_uv|`` of every removed vertex (an edge to a ground vertex), is
    walked ``samples`` times from both ends to the kept vertices, and the walks' endpoints get an
    edge of weight ``1 / (samples * sum of 1/w over the steps)``.  The expected result is the exact
    reduction; ``samples`` trades entries for variance (16: a spectrum within about +-12 % on
    k-NN graphs, with several times fewer entries than the exact level).  The draws come from
    Philox streams of ``seed`` (None means 0): the same seed gives the same bits.  The matrix
    must be symmetric with non-negative weights and diagonally dominant (excesses below
    ``-1e-12 M_uu`` raise ``ValueError``; smaller ones count as 0); a graph's weights are read
    from ``-offdiag(L)`` with no excess.  A walk longer than ``max_steps`` steps raises
    ``ValueError``.  The matrix branch then returns the sampled ``L_new`` with its diagonal.
    """
    from .graphs import Graph
    _check_kron_method(method, samples, max_steps)
    key = _sampling_seed(seed, 1 << 21)
    if isinstance(G, Graph):
        return _kron_graph(G, ind, method, int(samples), key, int(max_steps))
    _, dev = _ctx()
    M = _device_matrix(G, dev)
    _check_symmetric(M)
    ind = _kept_ids(ind, M.shape[0])
    if method == "walks":
        return _schur_walks(M, ind, int(samples), key, int(max_steps)).to_scipy().astype(np.float64)
    return _schur(M, ind).to_scipy().astype(np.float64)


def _laplacian_inverse(L):
    """(Ainv, labels, sizes) for a float64 Laplacian DeviceCSR: Ainv = (L + sum_c 1_c 1_c^T / |c|)^-1
    = L^+ + sum_c 1_c 1_c^T / |c| (dense, float64, on the device), by one Cholesky factor.
    labels: component of every vertex (smallest vertex id), sizes[v] = |component of v|."""
    torch = nat.require_cuda()
    n, dev = L.shape[0], L.device
    labels = torch.empty(n, dtype=torch.int32, device=dev)
    _call("gsp_cc_labels_f64", nat.i64(n), L.indptr, L.indices, L.data, nat.i32(0), labels, None)
    lab = labels.long()
    sizes = torch.bincount(lab, minlength=n)[lab].double()
    free, _ = torch.cuda.mem_get_info(dev)
    if 3 * n * n * 8 > free:
        raise ValueError("The dense factor of this {0} x {0} Laplacian needs about {1:.1f} GB of "
                         "device memory ({2:.1f} GB free).".format(n, 3 * n * n * 8 / 2 ** 30,
                                                                  free / 2 ** 30))
    A = L.to_dense()
    step = max(1, (1 << 26) // max(n, 1))
    for r0 in range(0, n, step):
        r1 = min(n, r0 + step)
        A[r0:r1] += (lab[r0:r1, None] == lab[None, :]) / sizes[r0:r1, None]
    C, info = torch.linalg.cholesky_ex(A)
    del A
    if int(info.item()) != 0:
        raise ValueError("The matrix is not a combinatorial Laplacian (its Cholesky factor "
                         "does not exist).")
    return torch.cholesky_inverse(C), lab, sizes


def resistance_distance(M):
    r"""Resistance distances of a graph (utils.py:140-181), a dense (N, N) float64 ndarray.

    ``M``: a :class:`Graph` with a combinatorial Laplacian, or a Laplacian as a sparse matrix.
    ``R_uv = L+_uu + L+_vv - 2 L+_uv`` with the pseudo-inverse ``L+`` from one float64 Cholesky
    factor of ``L + sum_c 1_c 1_c^T / |c|`` (one rank-one term per connected component), on the
    device.  The reference inverts the singular L with SuperLU and falls back to ``pinv`` only
    when SuperLU reports the singularity; this is exact.  Vertices of different components get
    ``L+_uu + L+_vv``, as with ``pinv``.
    """
    from .graphs import Graph
    torch, dev = _ctx()
    if isinstance(M, Graph):
        if M.lap_type != "combinatorial":
            raise ValueError("Need a combinatorial Laplacian.")
        dev, L = M.device, M.L
    else:
        L = M
    with torch.cuda.device(dev):
        Ainv, lab, sizes = _laplacian_inverse(_device_matrix(L, dev))
        n = Ainv.shape[0]
        step = max(1, (1 << 26) // max(n, 1))
        for r0 in range(0, n, step):
            r1 = min(n, r0 + step)
            Ainv[r0:r1] -= (lab[r0:r1, None] == lab[None, :]) / sizes[r0:r1, None]
        d = torch.diagonal(Ainv).clone()
        R = d[:, None] + d[None, :] - Ainv - Ainv.T
        return R.cpu().numpy()


def _sampling_seed(seed, i):
    return (int(0 if seed is None else seed) * 0x9E3779B97F4A7C15 + i) & 0xFFFFFFFFFFFFFFFF


# The resistance sketch (DESIGN.md section 4.22): CG stops at this relative residual per column,
# and its blocks of columns keep five (N, width) float64 arrays within this many bytes whatever
# the card, so that (seed, k, N) gives the same bits on any card.
_SKETCH_TOL = 1e-8
_SKETCH_BYTES = 32 << 30
_SKETCH_MAX_WIDTH = 256


def _sketch_dim(n, delta=0.5):
    """Default number of JL columns, ceil(24 ln N / delta^2) (at least 1)."""
    return max(1, int(np.ceil(24 * np.log(max(n, 1)) / delta ** 2)))


def _sketch_width(n, k):
    """Columns per CG block: min(k, 256, w_mem), w_mem the largest power of two >= 8 with
    5 * 8 * N * w_mem <= _SKETCH_BYTES; ValueError when even 8 columns do not fit."""
    if 5 * 8 * n * 8 > _SKETCH_BYTES:
        raise ValueError("The resistance sketch of this {0} x {0} Laplacian needs at least {1:.1f} "
                         "GB of device memory for a block of 8 columns (at most {2:.1f} GB are "
                         "used).".format(n, 5 * 8 * n * 8 / 2 ** 30, _SKETCH_BYTES / 2 ** 30))
    w = 8
    while w < _SKETCH_MAX_WIDTH and 5 * 8 * n * (2 * w) <= _SKETCH_BYTES:
        w *= 2
    return min(int(k), _SKETCH_MAX_WIDTH, w)


def _sketch_maxiter(n):
    """(CG iterations allowed per block, batches of 25 without halving the residual before CG
    gives up): 20 sqrt(N), at least 1000, and sqrt(N) / 25, at least 8.  A two-dimensional mesh
    of N vertices has a Jacobi-scaled condition number kappa that grows like N; CG needs about
    sqrt(kappa) / 3 iterations to halve its residual and a multiple of sqrt(kappa) to reach
    _SKETCH_TOL."""
    return int(max(1000, 20 * np.sqrt(n))), int(max(8, np.sqrt(n) / 25))


def _edge_resistances(Ld, start, end, k, seed):
    """Effective resistances of the edges (start[e], end[e]) of the float64 Laplacian DeviceCSR
    ``Ld`` by the Johnson-Lindenstrauss sketch with ``k`` columns (a float64 device tensor).

    R~_e = ||Z (chi_u - chi_v)||^2, Z = Q W^1/2 B L^+ / sqrt(k), Q the +-1 signs of
    gsp_jl_sketch_f64 from the Philox key ``_sampling_seed(seed, 1 << 20)``.  Per block of columns:
    the right-hand sides Y = D^-1/2 B^T W^1/2 Q^T / sqrt(k) on the device, block CG on the
    Jacobi-scaled Laplacian D^-1/2 L D^-1/2 (``learning._block_cg``), and the block's share of
    every R~_e with Z = D^-1/2 U.  Every column of Y is orthogonal to the null space D^1/2 1_c of a
    component, so the singular systems are consistent; the drift of the solution along that null
    space is a constant per component in Z, which cancels in Z_u - Z_v.  Blocks and columns are
    taken in order: the result is reproducible bit for bit.
    """
    import types
    from . import learning
    torch = nat.require_cuda()
    n, dev = Ld.shape[0], Ld.device
    width = _sketch_width(n, k)
    # D and the operator come from the weights alone: D = W 1 in float64 (row by row, in order)
    # and diag(Lhat) = 1, so that Lhat D^1/2 1_c = 0 to rounding.  A stored diagonal that is not
    # exactly W 1 (a float32 Laplacian) would make Lhat slightly indefinite, and CG diverge.
    rows, cols = row_ids(Ld.indptr), Ld.indices.long()
    off = rows != cols
    w = torch.where(off, -Ld.data, torch.zeros_like(Ld.data))
    deg = torch.empty(n, dtype=torch.float64, device=dev)
    _call("gsp_degree_f64", nat.i64(n), Ld.indptr, w, None, None, deg, None)
    dinv = torch.where(deg > 0, deg.clamp(min=1e-300).rsqrt(), torch.zeros_like(deg))
    diag = torch.nonzero(deg > 0).flatten()
    view = types.SimpleNamespace(L=DeviceCSR.from_coo(
        torch.cat([rows[off], diag]), torch.cat([cols[off], diag]),
        torch.cat([-dinv[rows[off]] * w[off] * dinv[cols[off]], torch.ones_like(deg[diag])]),
        Ld.shape))
    key = _sampling_seed(seed, 1 << 20)
    ne = int(start.numel())
    e32 = [x.to(torch.int32).contiguous() for x in (start, end)]
    R = torch.zeros(ne, dtype=torch.float64, device=dev)
    Y = torch.empty((n, width), dtype=torch.float64, device=dev)
    maxiter, patience = _sketch_maxiter(n)
    for j0 in range(0, k, width):
        wb = min(width, k - j0)
        Yb = Y if wb == width else torch.empty((n, wb), dtype=torch.float64, device=dev)
        _call("gsp_jl_sketch_f64", nat.i64(n), Ld.indptr, Ld.indices, Ld.data, dinv, nat.u64(key),
              nat.i64(j0), nat.i64(wb), nat.i64(k), Yb)
        U, _, _ = learning._block_cg(view, 1.0, None, None, Yb, _SKETCH_TOL, maxiter, patience)
        _call("gsp_jl_accumulate_f64", nat.i64(ne), e32[0], e32[1], U, dinv, nat.i64(wb), R)
        del U
    return R


def graph_sparsify(M, epsilon, maxiter=10, seed=None, *, resistances="exact", sketch_dim=None):
    r"""Sparsify a graph with Spielman-Srivastava (reduction.py:34-147).

    ``M``: a :class:`Graph` (combinatorial Laplacian, else ``NotImplementedError``) or a
    Laplacian as a sparse matrix; ``epsilon`` in ``[1/sqrt(N), 1)`` (else ``ValueError``).
    ``q = round(9 C^2 N log N / epsilon^2)`` edges are drawn with probability ``P_e`` proportional
    to ``w_e R_e`` (``R_e`` the edge's effective resistance, from one float64 Cholesky factor on
    the device), and an edge drawn ``k`` times gets the weight ``k w_e / (q P_e)``.  If the result
    is disconnected, epsilon is lowered and the sampling repeated, at most ``maxiter`` times.

    Differences from the reference (DESIGN.md section 2): the draws come from counter-based
    Philox streams of ``seed`` (``None`` means 0), so the same seed gives the same bits but not
    SciPy's draws; ``P_e`` is ``w_e R_e`` rounded to 32 bits relative to its largest value (the
    distribution actually sampled); per-edge counts stand for the removed ``stats.itemfreq``; the
    graph keeps its coordinates; a matrix in gives the Laplacian ``D' - W'`` as a SciPy CSR matrix
    out (the reference returns ``-W'`` as a ``lil_matrix``).

    ``resistances`` (an addition the reference does not have): ``'exact'`` (the default) as
    above, limited by the dense factor's 3 N^2 8 bytes to some 5 10^4 vertices; ``'sketch'``
    estimates every R_e by the Johnson-Lindenstrauss projection of Spielman-Srivastava, from
    ``sketch_dim`` = k Laplacian solves (default ``ceil(24 ln N / 0.5^2)``: every estimate within
    a factor 1 +- 0.5 with high probability, which is all the sampler needs).  The solves are
    block conjugate gradients on the Jacobi-scaled Laplacian in float64, in blocks of at most 256
    columns (DESIGN.md section 4.22); the signs come from Philox streams of ``seed``, so the same
    seed gives the same bits.  Everything after R_e is the same for both.  The sketch needs a
    symmetric Laplacian with non-negative weights (else ``ValueError``) and reads only its
    off-diagonal entries, the weights: the degrees are their row sums.
    """
    from .graphs import Graph
    if resistances not in ("exact", "sketch"):
        raise ValueError("resistances must be 'exact' or 'sketch', not {!r}.".format(resistances))
    if sketch_dim is not None and int(sketch_dim) < 1:
        raise ValueError("sketch_dim must be at least 1, not {}.".format(sketch_dim))
    torch, dev = _ctx()
    is_graph = isinstance(M, Graph)
    if is_graph:
        if not M.lap_type == "combinatorial":
            raise NotImplementedError
        dev, L, N = M.device, M.L, M.N
    else:
        L, N = M, np.shape(M)[0]
    if not 1.0 / np.sqrt(N) <= epsilon < 1:
        raise ValueError("GRAPH_SPARSIFY: Epsilon out of required range")

    with torch.cuda.device(dev):
        Ld = _device_matrix(L, dev)
        rows, cols = row_ids(Ld.indptr), Ld.indices.long()
        w = -Ld.data
        # edges: the lower triangle of W with w >= 1e-10 (reduction.py:89-97)
        edge = (rows > cols) & (w >= 1e-10)
        start, end, weights = rows[edge], cols[edge], w[edge].contiguous()
        ne = int(weights.numel())
        if resistances == "sketch":
            _check_symmetric(Ld, "The resistance sketch")
            if bool(((rows != cols) & (w < 0)).any()):
                raise ValueError("The resistance sketch needs non-negative edge weights (the "
                                 "Laplacian has a positive off-diagonal entry).")
            k = _sketch_dim(N) if sketch_dim is None else int(sketch_dim)
            R = _edge_resistances(Ld, start, end, k, seed)
        else:
            Ainv, _, _ = _laplacian_inverse(Ld)
            R = torch.empty(ne, dtype=torch.float64, device=dev)
            e32 = [x.to(torch.int32).contiguous() for x in (start, end)]
            _call("gsp_edge_resistance_f64", nat.i64(ne), e32[0], e32[1], Ainv, nat.i64(N), R)
            del Ainv
        x = weights * torch.clamp(R, min=0)
        xmax = float(x.max().item()) if ne else 0.0
        if not xmax > 0:
            raise ValueError("GRAPH_SPARSIFY: the graph has no edge with a positive weight")
        k = torch.round(x / xmax * 2.0 ** 32).to(torch.int64).contiguous()
        total = int(k.sum().item())
        Pe = k.double() / total
        counts = torch.empty(ne, dtype=torch.int64, device=dev)
        for i in range(maxiter):
            C0 = 1 / 30.0
            C = 4 * C0
            q = int(round(N * np.log(N) * 9 * C ** 2 / (epsilon ** 2)))
            _call("gsp_sparsify_sample", nat.i64(ne), k, nat.i64(q), nat.u64(_sampling_seed(seed, i)),
                  counts)
            hit = counts > 0
            new_w = counts[hit].double() * weights[hit] / (q * Pe[hit])
            r, c = start[hit], end[hit]
            sparser = Graph.from_coo(torch.cat([r, c]), torch.cat([c, r]), torch.cat([new_w, new_w]),
                                     N, dtype=torch.float64, device=dev)
            if sparser.is_connected():
                break
            elif i == maxiter - 1:
                logger.warning("Despite attempts to reduce epsilon, sparsified graph is "
                               "disconnected")
            else:
                epsilon -= (epsilon - 1 / np.sqrt(N)) / 2.0
        if is_graph:
            W = sparser.W
            return Graph(W, lap_type=M.lap_type, coords=getattr(M, "coords", None),
                         plotting=M.plotting, dtype=M.dtype, device=dev)
        sparser.compute_laplacian("combinatorial")
        return sparser.L.to_scipy().astype(np.float64)


def graph_multiresolution(G, levels, sparsify=True, sparsify_eps=None,
                          downsampling_method="largest_eigenvector", reduction_method="kron",
                          compute_full_eigen=False, reg_eps=0.005, *, seed=0,
                          kron_method="exact", kron_samples=16, resistances="exact"):
    r"""Compute a pyramid of graphs by Kron reduction (reduction.py:196-306).

    Per level: the eigenvector ``V`` of the largest eigenvalue of L (``G._largest_eigenvector``,
    on the device), ``V *= sign(V[0])``, keep ``ind = V >= 0``, Kron-reduce onto ``ind``
    (:func:`kron_reduction`), then, with ``sparsify``, :func:`graph_sparsify` with epsilon
    ``min(max(sparsify_eps, 2 / sqrt(N)), 1)``; then ``estimate_lmax()`` (or the full Fourier
    basis with ``compute_full_eigen``).  ``Gs[i + 1].mr = {'idx', 'orig_idx', 'level'}`` and, on
    the level above, ``mr['K_reg']`` (Kron reduction of ``L + reg_eps I``, a SciPy CSR matrix) and
    ``mr['green_kernel']``, as in the reference.  ``seed`` seeds the eigenvector solver and the
    sparsification of every level.

    Keyword-only additions: ``kron_method`` (``'exact'`` or ``'walks'``) and ``kron_samples`` select
    the reduction of every level and of ``mr['K_reg']`` (:func:`kron_reduction`'s ``method`` and
    ``samples``; the walks of level i are keyed from ``seed`` and i, those of its ``K_reg`` apart
    from them), and ``resistances`` is passed to :func:`graph_sparsify`.  With
    ``kron_method='walks', resistances='sketch'`` no step forms a dense block or factor, and the
    pyramid reaches graphs of 10^5 vertices and more (DESIGN.md section 4.23).  The synthesis
    still inverts the analysis exactly: both use the cached ``K_reg``.
    """
    _check_kron_method(kron_method, kron_samples)
    if resistances not in ("exact", "sketch"):
        raise ValueError("resistances must be 'exact' or 'sketch', not {!r}.".format(resistances))
    if sparsify_eps is None:
        sparsify_eps = min(10.0 / np.sqrt(G.N), 0.3)
    if compute_full_eigen:
        G.compute_fourier_basis()
    else:
        G.estimate_lmax()
    Gs = [G]
    Gs[0].mr = {"idx": np.arange(G.N), "orig_idx": np.arange(G.N)}
    for i in range(levels):
        if downsampling_method == "largest_eigenvector":
            V = Gs[i]._largest_eigenvector(seed=seed)
            V *= np.sign(V[0])
            ind = np.nonzero(V >= 0)[0]
        else:
            raise NotImplementedError("Unknown graph downsampling method.")
        if reduction_method == "kron":
            Gs.append(_kron_graph(Gs[i], ind, kron_method, int(kron_samples),
                                  _sampling_seed(seed, 2000 + i), _WALK_MAX_STEPS))
        else:
            raise NotImplementedError("Unknown graph reduction method.")
        if sparsify and Gs[i + 1].N > 2:
            Gs[i + 1] = graph_sparsify(Gs[i + 1], min(max(sparsify_eps, 2.0 / np.sqrt(Gs[i + 1].N)),
                                                      1.0), seed=_sampling_seed(seed, 1000 + i),
                                     resistances=resistances)
        if compute_full_eigen:
            Gs[i + 1].compute_fourier_basis()
        else:
            Gs[i + 1].estimate_lmax()
        Gs[i + 1].mr = {"idx": ind, "orig_idx": Gs[i].mr["orig_idx"][ind], "level": i}
        Gs[i].mr["K_reg"] = _kron_regularized(Gs[i], ind, reg_eps, kron_method, int(kron_samples),
                                              _sampling_seed(seed, 3000 + i))
        Gs[i].mr["_kreg_key"] = (reg_eps, ind.tobytes())
        Gs[i].mr["green_kernel"] = filters.Filter(Gs[i], lambda x: 1.0 / (reg_eps + x))
        Gs[i].mr["_green_eps"] = reg_eps
    return Gs


_TREE_METHODS = {"unweighted": 0, "sum": 1, "resistance_distance": 2}   # GSPB200_TREE_*
_TREE_MAX_N = 2 ** 30


def _tree_root(G, root):
    """(depth, parent, weight to parent) device tensors (int32, int32, float64) of the tree
    ``G._symmetric_adjacency()`` rooted at ``root`` (csrc/tree.cu).  ``ValueError`` when the
    graph is not connected or is not a tree."""
    torch = nat.require_cuda()
    n, dev = G.N, G.device
    if n > _TREE_MAX_N:
        raise ValueError("Tree multiresolution supports at most 2^30 vertices, not {}.".format(n))
    if not 0 <= root < n:
        raise ValueError("The root {} is not a vertex of the graph (N = {}).".format(root, n))
    Ws = G._symmetric_adjacency()
    with torch.cuda.device(dev):
        st = nat.stream_ptr(dev)
        # components of the symmetric adjacency: cc_labels reads the entries above the diagonal,
        # which a directed W need not store
        labels = torch.empty(n, dtype=torch.int32, device=dev)
        ncomp = torch.empty(1, dtype=torch.int64, device=dev)
        nat.call("gsp_cc_labels_" + G._sfx, nat.i64(n), Ws.indptr, Ws.indices, Ws.data, nat.i32(0),
                 labels, ncomp, st)
        arc_ptr = torch.empty(n + 1, dtype=torch.int32, device=dev)
        n_arcs = torch.empty(1, dtype=torch.int64, device=dev)
        nat.call("gsp_tree_arc_count", nat.i64(n), Ws.indptr, Ws.indices, arc_ptr, n_arcs, st)
        counts = torch.cat([ncomp, n_arcs]).cpu().numpy()
        if counts[0] != 1:
            raise ValueError("Graph is not connected")
        if counts[1] != 2 * (n - 1):
            raise ValueError("G must be a tree: a connected graph on {} vertices with {} edges "
                             "has {} off-diagonal entries, not {}.".format(
                                 n, n - 1, int(counts[1]), 2 * (n - 1)))
        depth = torch.empty(n, dtype=torch.int32, device=dev)
        parent = torch.empty(n, dtype=torch.int32, device=dev)
        wpar = torch.empty(n, dtype=torch.float64, device=dev)
        nat.call("gsp_tree_root_" + G._sfx, nat.i64(n), nat.i64(Ws.nnz), Ws.indptr, Ws.indices,
                 Ws.data, arc_ptr, nat.i32(root), depth, parent, wpar, st)
    return depth, parent, wpar


def _tree_depths(G, root):
    """(depth, parent) of every vertex of the tree G from ``root``, as int32 device tensors."""
    depth, parent, _ = _tree_root(G, int(root))
    return depth, parent


def _tree_level(G, depth, parent, wpar, root, method):
    """One coarsening of a rooted tree: (keep (host int64), Graph of the kept vertices, new root,
    and the next level's depth, parent and weight to parent)."""
    from .graphs import Graph
    torch = nat.require_cuda()
    n, dev = int(depth.numel()), G.device
    with torch.cuda.device(dev):
        st = nat.stream_ptr(dev)
        new_id = torch.empty(n + 1, dtype=torch.int32, device=dev)
        n_new_dev = torch.empty(1, dtype=torch.int64, device=dev)
        nat.call("gsp_tree_keep", nat.i64(n), depth, new_id, n_new_dev, st)
        n_new = int(n_new_dev.item())
        m = 2 * (n_new - 1)
        keep = torch.empty(n_new, dtype=torch.int64, device=dev)
        rows = torch.empty(m, dtype=torch.int32, device=dev)
        cols = torch.empty(m, dtype=torch.int32, device=dev)
        vals = torch.empty(m, dtype=G.dtype, device=dev)
        new_depth = torch.empty(n_new, dtype=torch.int32, device=dev)
        new_parent = torch.empty(n_new, dtype=torch.int32, device=dev)
        new_wpar = torch.empty(n_new, dtype=torch.float64, device=dev)
        nat.call("gsp_tree_coarsen_" + G._sfx, nat.i64(n), nat.i64(n_new), depth, parent, wpar,
                 new_id, nat.i32(root), nat.i32(_TREE_METHODS[method]), keep, rows, cols, vals,
                 new_depth, new_parent, new_wpar, st)
        keep_host = keep.cpu().numpy()
        new_root = int(np.searchsorted(keep_host, root))
        W = DeviceCSR.from_coo(rows, cols, vals, (n_new, n_new))
    Gn = Graph(W, lap_type=G.lap_type, coords=G.coords[keep_host] if hasattr(G, "coords") else None,
               plotting=G.plotting, dtype=G.dtype, device=dev)
    Gn.root = new_root
    return keep_host, Gn, new_root, new_depth, new_parent, new_wpar


def tree_multiresolution(G, Nlevel, reduction_method="resistance_distance",
                         compute_full_eigen=False, root=None):
    r"""Compute a multiresolution of trees (reduction.py:633-787).

    ``G`` must be a tree: its symmetric adjacency (W, or (W + W^T) / 2 when directed; self-loops
    ignored) is connected with 2 (N - 1) off-diagonal entries, else ``ValueError``.  ``root``:
    ``G.root`` when None and G has one, else 1; an explicit 0 is honoured.  Per level, the
    vertices of even depth are kept (in increasing order), and every kept vertex other than the
    root is joined to its grandparent by an edge whose weight combines the weights w(v) to the
    parent and w(p) from the parent to the grandparent: 1 (``'unweighted'``), w(v) + w(p)
    (``'sum'``) or 1 / (1 / w(v) + 1 / w(p)) (``'resistance_distance'``), in float64, rounded once
    to ``G.dtype``.  Depths are halved, the root keeps its place.

    The tree is rooted on the device by an Euler tour ranked by pointer jumping, in O(log N)
    launches whatever its depth, and each level is a few O(N) kernels (csrc/tree.cu; DESIGN.md
    section 4.21).  Returns ``(Gs, subsampled_vertex_indices)``: ``Gs[0] is G`` and ``Nlevel``
    coarser graphs (each with ``root``, the level's coordinates, ``lap_type`` and ``dtype`` of G,
    and ``mr = {'idx', 'orig_idx', 'level'}`` as :func:`graph_multiresolution` sets, so
    :func:`pyramid_analysis` and :func:`pyramid_synthesis` run on the pyramid), and the
    ``Nlevel`` ascending int64 arrays of the kept vertices.  ``compute_full_eigen`` computes the
    Fourier basis of every level, ``Gs[0]`` included.  A level of one vertex has no edge; the
    levels after it repeat it.
    """
    if reduction_method not in _TREE_METHODS:
        raise ValueError("Unknown graph reduction method.")
    if root is None:
        root = getattr(G, "root", 1)
    root = int(root)
    depth, parent, wpar = _tree_root(G, root)
    if compute_full_eigen:
        G.compute_fourier_basis()
    Gs = [G]
    G.mr = {"idx": np.arange(G.N), "orig_idx": np.arange(G.N)}
    subsampled_vertex_indices = []
    for lev in range(Nlevel):
        keep, Gn, root, depth, parent, wpar = _tree_level(Gs[lev], depth, parent, wpar, root,
                                                          reduction_method)
        Gn.mr = {"idx": keep, "orig_idx": Gs[lev].mr["orig_idx"][keep], "level": lev}
        if compute_full_eigen:
            Gn.compute_fourier_basis()
        Gs.append(Gn)
        subsampled_vertex_indices.append(keep)
    return Gs, subsampled_vertex_indices


def _kron_regularized(G, ind, reg_eps, method="exact", samples=16, key=0):
    """Kron reduction of L + reg_eps I onto ind (reduction.py:302-303), L + reg_eps I assembled
    on the device.  ``method='walks'`` samples it with the Philox key ``key``, the excess of every
    vertex being reg_eps itself (not re-derived from the assembled diagonal)."""
    torch = nat.require_cuda()
    with torch.cuda.device(G.device):
        L = _device_matrix(G.L, G.device)
        n = G.N
        diag = torch.arange(n, dtype=torch.int32, device=G.device)
        M = DeviceCSR.from_coo(torch.cat([row_ids(L.indptr).to(torch.int32), diag]),
                               torch.cat([L.indices, diag]),
                               torch.cat([L.data, torch.full((n,), float(reg_eps),
                                                             dtype=torch.float64,
                                                             device=G.device)]), (n, n))
        if method == "walks":
            excess = torch.full((n,), float(reg_eps), dtype=torch.float64, device=G.device)
            return _schur_walks(M, ind, samples, key, _WALK_MAX_STEPS,
                                excess=excess).to_scipy().astype(np.float64)
        return _schur(M, ind).to_scipy().astype(np.float64)


def _as_columns(s):
    s = np.asarray(s) if not hasattr(s, "is_cuda") else s
    return s.reshape(s.shape[0], -1)


def _filter_columns(g, block, **kwargs):
    """One-filter bank applied to every column of an (N, Nv) block -> (N, Nv)."""
    out = g.filter(block if block.shape[1] > 1 else block[:, 0], **kwargs)
    return out.reshape(block.shape)


def _level_operator(G, reg_eps):
    """(K_reg, Green filter) of a level; cached in G.mr like graph_multiresolution does."""
    mr = getattr(G, "mr", None)
    if mr is None:
        mr = G.mr = {}
    if "green_kernel" not in mr or mr.get("_green_eps") != reg_eps:
        mr["green_kernel"] = filters.Filter(G, lambda x: 1.0 / (reg_eps + x))
        mr["_green_eps"] = reg_eps
    return mr


def interpolate(G, f_subsampled, keep_inds, order=100, reg_eps=0.005, **kwargs):
    r"""Interpolate a graph signal from its samples on ``keep_inds`` (reduction.py:150-193).

    ``alpha = K_reg f`` with ``K_reg`` the Kron reduction of ``L + eps I`` onto the samples
    (taken from ``G.mr['K_reg']`` when the multiresolution set-up stored it), zero-fill, then
    the Green kernel ``1 / (eps + x)`` as an order-``order`` Chebyshev filter on the device.
    Returns (N, Nv).
    """
    keep_inds = np.asarray(keep_inds)
    mr = _level_operator(G, reg_eps)
    K_reg = mr.get("K_reg")
    if K_reg is None or mr.get("_kreg_key") not in (None, (reg_eps, keep_inds.tobytes())):
        K_reg = kron_reduction(G.L.to_scipy().astype(np.float64) + reg_eps * sparse.eye(G.N),
                               keep_inds)
        mr["K_reg"], mr["_kreg_key"] = K_reg, (reg_eps, keep_inds.tobytes())
    sub = _as_columns(np.asarray(f_subsampled, dtype=np.float64))
    if sub.shape[0] != keep_inds.size:
        raise ValueError("f_subsampled must have one row per kept vertex")
    full = np.zeros((G.N, sub.shape[1]))
    full[keep_inds] = K_reg.dot(sub)
    return _filter_columns(mr["green_kernel"], full, order=order, **kwargs)


def _level_filters(h_filters, levels):
    if not isinstance(h_filters, list):
        if callable(h_filters):
            logger.warning("Converting filters into a list.")
            h_filters = [h_filters]
        else:
            raise TypeError("Filters must be a list of functions.")
    if len(h_filters) == 1:
        h_filters = h_filters * levels
    elif len(h_filters) != levels:
        raise ValueError("The number of filters must be one or equal to {}.".format(levels))
    return h_filters


def pyramid_analysis(Gs, f, **kwargs):
    r"""Graph pyramid transform (reduction.py:384-449).

    Per level: low-pass ``h(L) ca_i`` (Chebyshev filter on the device), keep the vertices
    of the next level, interpolate them back (:func:`interpolate`), prediction error
    ``pe_i = ca_i - interpolation``.  ``h_filters``: list of kernels (default
    ``1 / (2x + 1)``); remaining keyword arguments (``order`` ...) go to the filters, as in the
    reference.  Returns ``(ca, pe)``: lists of (n_level, Nv) arrays.
    """
    f = np.asarray(f)
    if f.shape[0] != Gs[0].N:
        raise ValueError("PYRAMID ANALYSIS: The signal to analyze should have the same "
                         "dimension as the first graph.")
    levels = len(Gs) - 1
    h_filters = _level_filters(kwargs.pop("h_filters", lambda x: 1.0 / (2 * x + 1)), levels)
    ca, pe = [_as_columns(f.astype(np.float64))], []
    for i in range(levels):
        idx = np.asarray(Gs[i + 1].mr["idx"])
        s_low = _filter_columns(filters.Filter(Gs[i], h_filters[i]), ca[i], **kwargs)
        ca.append(s_low[idx])
        s_pred = interpolate(Gs[i], ca[i + 1], idx, **kwargs)
        pe.append(ca[i] - s_pred)
    return ca, pe


def pyramid_synthesis(Gs, cap, pe, order=30, **kwargs):
    r"""Signal from its pyramid coefficients, direct method (reduction.py:452-532).

    From the coarsest approximation up: interpolate to the finer level (order-``order`` Green
    kernel filter on the device) and add that level's prediction error.  Returns
    ``(reconstruction, ca)``.
    """
    if bool(kwargs.pop("least_squares", False)):
        raise NotImplementedError(
            "least-squares pyramid synthesis is broken in the reference (reduction.py:593) and "
            "is not part of this engine; use the direct method.")
    kwargs.pop("use_landweber", None)
    reg_eps = float(kwargs.pop("reg_eps", 0.005))
    levels = len(Gs) - 1
    if len(pe) != levels:
        raise ValueError("Gs and pe have different shapes.")
    ca = [_as_columns(np.asarray(cap, dtype=np.float64))]
    for i in range(levels):
        lv = levels - i - 1
        s_pred = interpolate(Gs[lv], ca[i], np.asarray(Gs[lv + 1].mr["idx"]), order=order,
                             reg_eps=reg_eps, **kwargs)
        ca.append(s_pred + _as_columns(np.asarray(pe[lv])))
    return ca[levels], ca
