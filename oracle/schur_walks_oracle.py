"""NumPy restatement of ``kron_reduction(method='walks')`` (pygsp_b200/reduction.py
``_schur_walks``, csrc/schur_walk.cu), and the dense exact Schur complement it estimates.

Test infrastructure: nothing under pygsp_b200/ imports this module.

The sampler is the random-walk Schur complement of Durfee, Kyng, Peebles, Rao and Sachdeva
(STOC 2017).  M is an SDDM matrix: weights w_uv = -M_uv and an excess e_u = M_uu - sum_v w_uv,
an edge (u, g) to a ground vertex.  Every item walks from one end of an edge until it hits a kept
vertex or g, then from the other end; the rule, the draws and the float64 operation order are the
device's, vectorised over the items, so the same key gives the same samples bit for bit:

* step t of item i (counted over both walks) reads words 2 (t mod 2), 2 (t mod 2) + 1 (lo, hi) of
  ``curand4(key, i, t div 2)`` and U = (((hi << 32) | lo) >> 11) 2^-53;
* at x, X = U (total_x + e_x): ground when X >= total_x and e_x > 0, else the first entry of the
  row whose inclusive prefix of weights exceeds X (the last positive weight when none does);
* R = (steps of the first walk) + 1/w + (steps of the second), summed in that order, and the
  sample's value is 1 / (R samples).

* ``prep``        -- prefix sums, row totals and excesses, with the device's error flags.
* ``walk_items``  -- the endpoints, values and step counts of every item.
* ``schur_walks`` -- the sampled reduction as a SciPy CSR matrix in the order of ``ind``.
* ``dense_schur`` -- SC(M, K) in float64, dense, without the components that have no kept
  neighbour (they contribute nothing).
"""
import numpy as np
from scipy import sparse
from scipy.sparse import csgraph

from oracle.random_graphs_oracle import curand4

GROUND, CAPPED = -1, -2


def _canonical(M):
    M = sparse.csr_matrix(M, dtype=np.float64)
    M.sum_duplicates()
    M.eliminate_zeros()
    M.sort_indices()
    return M


def prep(M, excess=None):
    """(prefix, total, excess, flags) of gsp_walk_prep_f64: flags bit 1 for a positive
    off-diagonal entry, bit 2 (derived excess only) for an excess below -1e-12 M_uu."""
    M = _canonical(M)
    n = M.shape[0]
    rows = np.repeat(np.arange(n), np.diff(M.indptr))
    off = rows != M.indices
    w = np.where(off, -M.data, 0.0)
    prefix = np.empty_like(w)
    total = np.zeros(n)
    for u in range(n):                        # sequential per row, in CSR order
        acc = 0.0
        for k in range(M.indptr[u], M.indptr[u + 1]):
            acc += w[k]
            prefix[k] = acc
        total[u] = acc
    flags = 1 if bool((M.data[off] > 0).any()) else 0
    if excess is None:
        diag = M.diagonal()
        ex = diag - total
        if bool((ex < -1e-12 * diag).any()):
            flags |= 2
    else:
        ex = np.broadcast_to(np.asarray(excess, dtype=np.float64), (n,)).copy()
    return prefix, total, np.maximum(ex, 0.0), flags


def split(M, ind):
    """(slot, dead) of the kept vertices ``ind``: slot[v] = -1 - (index of v in ind) for a kept
    vertex and 0 for a removed one; dead[v] for a removed vertex whose component of the removed
    vertices has no kept neighbour."""
    M = _canonical(M)
    n = M.shape[0]
    ind = np.asarray(ind, dtype=np.int64)
    slot = np.zeros(n, dtype=np.int64)
    slot[ind] = -1 - np.arange(ind.size)
    rem = np.flatnonzero(slot == 0)
    dead = np.zeros(n, dtype=bool)
    if rem.size:
        S = M[rem][:, rem]
        nc, lab = csgraph.connected_components(S, directed=False)
        rows = np.repeat(np.arange(n), np.diff(M.indptr))
        comp = np.full(n, -1)
        comp[rem] = lab
        touch = (comp[rows] >= 0) & (slot[M.indices] < 0)
        has = np.zeros(nc, dtype=bool)
        has[comp[rows[touch]]] = True
        dead[rem] = ~has[lab]
    return slot, dead


def items(M, ind, excess=None):
    """(eu, ev, ew, gu): the sampled edges (u > v, lower triangle in CSR order, at least one end
    removed, not dead) and the removed live vertices with a positive excess, ascending."""
    M = _canonical(M)
    n = M.shape[0]
    slot, dead = split(M, ind)
    _, _, ex, _ = prep(M, excess)
    rows = np.repeat(np.arange(n), np.diff(M.indptr))
    cols = M.indices.astype(np.int64)
    e = (rows > cols) & ((slot[rows] >= 0) | (slot[cols] >= 0)) & ~dead[rows]
    gu = np.flatnonzero((slot >= 0) & ~dead & (ex > 0))
    return rows[e], cols[e], -M.data[e], gu


def _uniform(key, item, t):
    words = curand4(key, item.astype(np.uint64), (t // 2).astype(np.uint64))
    odd = (t & 1).astype(bool)
    lo = np.where(odd, words[2], words[0])
    hi = np.where(odd, words[3], words[1])
    return ((hi << np.uint64(32)) | lo) >> np.uint64(11)


def _walk(M, prefix, total, ex, slot, key, item, x, R, t, max_steps):
    """Walk every item from x until a kept vertex, the ground or max_steps; R and t are updated
    in place.  Returns the kept index, GROUND or CAPPED of every item."""
    out = np.full(x.size, CAPPED, dtype=np.int64)
    act = np.arange(x.size)
    x = x.copy()
    while act.size:
        s = slot[x[act]]
        kept = s < 0
        out[act[kept]] = -1 - s[kept]
        act = act[~kept]
        capped = t[act] >= max_steps
        act = act[~capped]
        if not act.size:
            break
        xa = x[act]
        U = _uniform(key, item[act], t[act]).astype(np.float64) * 2.0 ** -53
        t[act] += 1
        tot, e = total[xa], ex[xa]
        X = U * (tot + e)
        g = (X >= tot) & (e > 0)
        R[act[g]] += 1.0 / e[g]
        out[act[g]] = GROUND
        act, xa, X, tot = act[~g], xa[~g], X[~g], tot[~g]
        lo, hi = M.indptr[xa].astype(np.int64), M.indptr[xa + 1].astype(np.int64)
        p = _search(prefix, lo, hi, X, strict=True)
        none = p == hi
        if none.any():
            p[none] = _search(prefix, lo[none], hi[none], tot[none], strict=False)
        R[act] += 1.0 / -M.data[p]
        x[act] = M.indices[p]
    return out


def _search(prefix, lo, hi, x, strict):
    lo, hi = lo.copy(), hi.copy()
    while True:
        open_ = lo < hi
        if not open_.any():
            return lo
        mid = lo + ((hi - lo) >> 1)
        p = prefix[np.where(open_, mid, 0)]
        right = (p > x) if strict else (p >= x)
        hi = np.where(open_ & right, mid, hi)
        lo = np.where(open_ & ~right, mid + 1, lo)


def walk_items(M, ind, samples, key, excess=None, max_steps=2 ** 20):
    """Every item of the device's launch: dict of item ids, (c1, c2) (kept index or GROUND;
    CAPPED when max_steps stopped it), val = 1 / (R samples) and steps."""
    M = _canonical(M)
    prefix, total, ex, _ = prep(M, excess)
    slot, _ = split(M, ind)
    eu, ev, ew, gu = items(M, ind, excess)
    ne, ng = eu.size * samples, gu.size * samples
    item = np.arange(ne + ng, dtype=np.int64)
    a = np.concatenate([np.repeat(eu, samples), np.repeat(gu, samples)])
    inv_w = np.concatenate([1.0 / np.repeat(ew, samples), 1.0 / ex[np.repeat(gu, samples)]])
    R = np.zeros(item.size)
    t = np.zeros(item.size, dtype=np.int64)
    c1 = _walk(M, prefix, total, ex, slot, key, item, a, R, t, max_steps)
    ok = c1 != CAPPED
    R[ok] += inv_w[ok]
    c2 = np.full(item.size, GROUND, dtype=np.int64)
    e = ok & (item < ne)
    if e.any():
        b = np.repeat(ev, samples)[e[:ne]]
        Re, te = R[e], t[e]
        c2[e] = _walk(M, prefix, total, ex, slot, key, item[e], b, Re, te, max_steps)
        R[e], t[e] = Re, te
    return {"item": item, "edge": item < ne, "c1": c1, "c2": c2,
            "val": 1.0 / (R * float(samples)), "steps": t}


def triplets(res):
    """(rows, cols, vals) the items emit, in item order (empty slots left out)."""
    r, c, v = [], [], []
    c1, c2, val = res["c1"], res["c2"], res["val"]
    live = (c1 != CAPPED) & (c2 != CAPPED) & (c1 != c2)
    for i in np.flatnonzero(live):
        if c1[i] == GROUND or c2[i] == GROUND:
            k = c2[i] if c1[i] == GROUND else c1[i]
            r.append(k), c.append(k), v.append(val[i])
        else:
            r += [c1[i], c2[i], c1[i], c2[i]]
            c += [c2[i], c1[i], c1[i], c2[i]]
            v += [-val[i], -val[i], val[i], val[i]]
    return np.array(r, dtype=np.int64), np.array(c, dtype=np.int64), np.array(v)


def exact_part(M, ind, excess=None):
    """(rows, cols, vals) of the exact samples in the device's emission order: every kept-kept
    entry (rows in the order of ``ind``, each row's entries in M's column order), then its
    diagonal share -M_uv at (u, u) in the same order, then the excess of every kept vertex."""
    M = _canonical(M)
    ind = np.asarray(ind, dtype=np.int64)
    slot, _ = split(M, ind)
    _, _, ex, _ = prep(M, excess)
    Mk = M[ind].tocoo()                         # row slicing keeps each row's column order
    col = -1 - slot[Mk.col]
    e = (slot[Mk.col] < 0) & (col != Mk.row)
    r, c, v = Mk.row[e].astype(np.int64), col[e], Mk.data[e]
    kx = np.flatnonzero(ex[ind] > 0)
    return (np.concatenate([r, r, kx]), np.concatenate([c, r, kx]),
            np.concatenate([v, -v, ex[ind][kx]]))


def sum_in_order(rows, cols, vals, shape):
    """CSR of COO triplets, the values of one (row, col) added one after the other in the order
    given (the arithmetic of DeviceCSR.from_coo)."""
    order = np.lexsort((cols, rows))
    r, c, v = rows[order], cols[order], vals[order]
    first = np.r_[True, (r[1:] != r[:-1]) | (c[1:] != c[:-1])] if r.size else np.zeros(0, bool)
    start = np.flatnonzero(first)
    size = np.diff(np.r_[start, r.size])
    acc = v[start].copy()
    for k in range(1, int(size.max()) if size.size else 0):
        g = size > k
        acc[g] += v[start[g] + k]
    return sparse.csr_matrix((acc, (r[start], c[start])), shape=shape)


def schur_walks(M, ind, samples, key, excess=None, max_steps=2 ** 20):
    """The sampled reduction (m x m SciPy CSR, float64) in the order of ``ind``: M[ind][:, ind]
    when nothing is removed, else the exact samples then every item's, summed in that order."""
    M = _canonical(M)
    ind = np.asarray(ind, dtype=np.int64)
    m = ind.size
    if m == M.shape[0]:
        return M[ind][:, ind].tocsr()
    r0, c0, v0 = exact_part(M, ind, excess)
    r1, c1, v1 = triplets(walk_items(M, ind, samples, key, excess, max_steps))
    return sum_in_order(np.concatenate([r0, r1]), np.concatenate([c0, c1]),
                        np.concatenate([v0, v1]), (m, m))


def dense_schur(M, ind):
    """SC(M, K) = M_KK - M_KS M_SS^-1 M_SK (dense float64) over the live removed vertices."""
    M = _canonical(M)
    ind = np.asarray(ind, dtype=np.int64)
    slot, dead = split(M, ind)
    S = np.flatnonzero((slot >= 0) & ~dead)
    A = M.toarray()
    out = A[np.ix_(ind, ind)]
    if S.size:
        out = out - A[np.ix_(ind, S)] @ np.linalg.solve(A[np.ix_(S, S)], A[np.ix_(S, ind)])
    return out


def generalized_spread(LH, SC, tol=1e-9):
    """(min, max) of the generalised eigenvalues of (LH, SC) on the range of SC."""
    lam, V = np.linalg.eigh(SC)
    keep = lam > tol * lam.max()
    P = V[:, keep] / np.sqrt(lam[keep])
    mu = np.linalg.eigvalsh(P.T @ LH @ P)
    return float(mu.min()), float(mu.max())


def knn_laplacian(n, k=10, seed=0):
    """Combinatorial Laplacian (SciPy CSR) of a uniformly random 2-D k-NN graph with Gaussian
    weights exp(-d^2 / sigma^2), sigma the mean neighbour distance, symmetrised by the maximum."""
    from scipy.spatial import cKDTree
    pts = np.random.default_rng(seed).uniform(size=(n, 2))
    d, j = cKDTree(pts).query(pts, k + 1)
    d, j = d[:, 1:], j[:, 1:]
    sigma = d.mean()
    W = sparse.csr_matrix((np.exp(-(d / sigma) ** 2).ravel(), (np.repeat(np.arange(n), k),
                                                               j.ravel())), shape=(n, n))
    W = W.maximum(W.T)
    return (sparse.diags(np.asarray(W.sum(axis=1)).ravel()) - W).tocsr()


def eigenvector_split(L):
    """Kept vertices of graph_multiresolution's split: the sign of the largest eigenvector."""
    _, V = np.linalg.eigh(L.toarray())
    v = V[:, -1] * np.sign(V[0, -1])
    return np.flatnonzero(v >= 0)
