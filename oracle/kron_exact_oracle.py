"""Host restatements of the exact Kron reduction's pieces (csrc/schur.cu and pygsp_b200/reduction.py
_split, _removed_components, _schur) and of the Spielman-Srivastava sampler gsp_sparsify_sample.

Test infrastructure: nothing under pygsp_b200/ imports this module.

* ``build_components`` -- a symmetric float64 Laplacian-like matrix M and kept vertices ``ind``
  whose removed vertices form exactly the requested components: each of a given size s, joined to
  exactly b distinct kept vertices, and well-conditioned, ill-conditioned or indefinite.
* ``removed_components`` -- the connected components of the removed vertices from SciPy, in the
  device's order (increasing smallest vertex), each with its kept neighbours in kept-index order.
* ``schur_blocks`` -- every component's block -M_BS M_SS^-1 M_SB by a dense float64 solve, with
  kappa_2(M_SS), and ``schur_tolerance``, the per-entry error bound built from them.
* ``sparsify_counts`` -- every draw of gsp_sparsify_sample replayed from Philox4x32-10 and the
  cumulative table of the integer weights, with Python integers for the 128-bit product.
"""
import numpy as np
from scipy import sparse
from scipy.sparse import csgraph

from .random_graphs_oracle import curand4

KINDS = ("well", "ill", "indefinite")
DRAWS_PER_CHUNK = 128      # kDrawsPerChunk of csrc/schur.cu: draw d belongs to chunk d // 128


def build_components(specs, n_kept=None, seed=0):
    """(M, ind, comps) for the removed components ``specs``, a list of (s, b, kind).

    Vertex ids mix kept and removed vertices at random, but the smallest vertex of component c
    increases with c, so the components come out in the order of ``specs``.  Each component is a
    path over its vertices in random order plus s // 2 random chords, and is joined to b distinct
    kept vertices drawn from one pool, so the kept neighbours of different components interleave;
    some kept vertices are also joined to each other.  ``ind`` lists the kept vertices in random
    order.  Kinds (s >= 2 for the last two):

    * ``'well'``: weights in [0.5, 1.5] and an excess in [1, 2] on every removed diagonal entry:
      kappa_2(M_SS) is at most a few tens, and M_SS is positive definite even when b = 0;
    * ``'ill'``: weights from 1e-6 to 1, no excess: a core of weights 10^U(-1, 0) carries the
      chords and the kept neighbours (weights 10^U(-6, 0)), and a tail path of weights
      10^U(-6, -5) hangs off it, whose slowest mode, about 1e-6 (2 / s)^2, sets
      lambda_min(M_SS): kappa_2(M_SS) is above 1e6 from s = 8, near 1e8 from s = 16 and 1e9 at
      s = 64, smaller for s <= 3;
    * ``'indefinite'``: the weights of 'well', and a removed diagonal of a tenth of the entry's
      weights inside the component: every pivot starts positive, 1^T M_SS 1 < 0.

    ``comps[c]`` = dict(vertices (ascending ids), kept (kept indices, ascending), s, b, kind).
    Kept vertices have the diagonal (weight sum) + 1.
    """
    rng = np.random.default_rng(seed)
    specs = [(int(s), int(b), str(kind)) for s, b, kind in specs]
    for s, b, kind in specs:
        if kind not in KINDS or s < 1 or b < 0 or (kind != "well" and s < 2):
            raise ValueError("bad component spec {}".format((s, b, kind)))
    nc = len(specs)
    bmax = max([b for _, b, _ in specs] + [1])
    n_kept = max(bmax + bmax // 4, 2 * nc, 8) if n_kept is None else int(n_kept)
    if n_kept < bmax:
        raise ValueError("fewer kept vertices than kept neighbours")
    nr = sum(s for s, _, _ in specs)
    n = nr + n_kept

    # ids by sorting keys: component c's first vertex has the c-th smallest anchor and its other
    # vertices larger keys, so its smallest id comes from the anchor
    anchors = np.sort(rng.uniform(0.0, 1.0, nc))
    keys, starts, pos = np.empty(n), [], 0
    for c, (s, _, _) in enumerate(specs):
        starts.append(pos)
        keys[pos] = anchors[c]
        keys[pos + 1:pos + s] = rng.uniform(anchors[c], 1.0, s - 1)
        pos += s
    keys[nr:] = rng.uniform(0.0, 1.0, n_kept)
    vid = np.empty(n, dtype=np.int64)
    vid[np.argsort(keys, kind="stable")] = np.arange(n)
    kept_ids = vid[nr:]
    ind = rng.permutation(kept_ids)
    kept_index = np.full(n, -1, dtype=np.int64)
    kept_index[ind] = np.arange(n_kept)

    rows, cols, vals = [], [], []
    excess = np.zeros(n)
    inner = np.zeros(n)          # weight of each removed vertex's edges inside its component
    kinds = np.array([""] * n, dtype=object)
    comps = []

    for c, (s, b, kind) in enumerate(specs):
        v = vid[starts[c]:starts[c] + s]
        kinds[v] = kind
        order = rng.permutation(v)
        # chords and kept neighbours touch order[:core] only; for 'ill' the rest is the tail
        core = (s + 1) // 2 if kind == "ill" else s
        a = list(order[:-1])
        z = list(order[1:])
        if kind == "ill":
            w = np.where(np.arange(s - 1) < core - 1, 10.0 ** rng.uniform(-1.0, 0.0, s - 1),
                         10.0 ** rng.uniform(-6.0, -5.0, s - 1))
        else:
            w = rng.uniform(0.5, 1.5, s - 1)
        if core >= 3:
            for _ in range(s // 2):
                i, j = rng.choice(core, 2, replace=False)
                a.append(order[i])
                z.append(order[j])
            w = np.r_[w, 10.0 ** rng.uniform(-1.0, 0.0, s // 2) if kind == "ill"
                      else rng.uniform(0.5, 1.5, s // 2)]
        rows += a
        cols += z
        vals += list(w)
        np.add.at(inner, a, w)
        np.add.at(inner, z, w)
        nbr = rng.choice(kept_ids, b, replace=False) if b else np.zeros(0, dtype=np.int64)
        extra = rng.random(b) < 0.5                   # some kept vertices get a second edge
        ka = list(nbr) + list(nbr[extra])
        kz = list(order[rng.integers(0, core, len(ka))])
        rows += ka
        cols += kz
        vals += list(10.0 ** rng.uniform(-6.0, 0.0, len(ka)) if kind == "ill"
                     else rng.uniform(0.5, 1.5, len(ka)))
        if kind == "well":
            excess[v] = rng.uniform(1.0, 2.0, s)
        comps.append(dict(vertices=np.sort(v), kept=np.sort(kept_index[nbr]), s=s, b=b,
                          kind=kind))
    for _ in range(n_kept):
        i, j = rng.choice(kept_ids, 2, replace=False)
        rows.append(i)
        cols.append(j)
        vals.append(rng.uniform(0.5, 1.5))

    W = sparse.coo_matrix((vals, (rows, cols)), shape=(n, n)).tocsr()
    W = (W + W.T).tocsr()
    W.sum_duplicates()
    deg = np.asarray(W.sum(axis=1)).ravel()
    diag = deg + excess
    diag[kept_ids] = deg[kept_ids] + 1.0
    bad = kinds == "indefinite"
    diag[bad] = 0.1 * inner[bad]
    M = (sparse.diags(diag) - W).tocsr()
    M.sum_duplicates()
    M.eliminate_zeros()
    M.sort_indices()
    return M, ind.astype(np.int64), comps


def removed_components(M, ind):
    """Components of the vertices not in ``ind``, joined by M's stored off-diagonal entries, from
    SciPy: a list of dict(vertices (ascending), kept (kept indices of the neighbours,
    ascending)), ordered by smallest vertex as gsp_component_order numbers them."""
    M = sparse.csr_matrix(M, dtype=np.float64)
    M.eliminate_zeros()
    n = M.shape[0]
    ind = np.asarray(ind, dtype=np.int64)
    kept_index = np.full(n, -1, dtype=np.int64)
    kept_index[ind] = np.arange(ind.size)
    rem = np.flatnonzero(kept_index < 0)
    if rem.size == 0:
        return []
    nc, lab = csgraph.connected_components(M[rem][:, rem], directed=False)
    first = np.full(nc, n, dtype=np.int64)
    np.minimum.at(first, lab, rem)
    rank = np.empty(nc, dtype=np.int64)
    rank[np.argsort(first)] = np.arange(nc)
    comp = np.full(n, -1, dtype=np.int64)
    comp[rem] = rank[lab]
    C = M.tocoo()
    hit = (comp[C.row] >= 0) & (kept_index[C.col] >= 0)
    pairs = np.unique(np.stack([comp[C.row[hit]], kept_index[C.col[hit]]], axis=1), axis=0)
    out = []
    for c in range(nc):
        out.append(dict(vertices=np.sort(np.flatnonzero(comp == c)),
                        kept=pairs[pairs[:, 0] == c, 1] if pairs.size else np.zeros(0, np.int64)))
    return out


def schur_blocks(M, ind, comps=None):
    """For every component of ``removed_components(M, ind)`` (or ``comps``): dict(vertices, kept,
    block = -M_BS solve(M_SS, M_SB) as a b x b float64 array with B in kept-index order,
    kappa = kappa_2(M_SS)).  A component without kept neighbours gets an empty block."""
    M = sparse.csr_matrix(M, dtype=np.float64)
    ind = np.asarray(ind, dtype=np.int64)
    comps = removed_components(M, ind) if comps is None else comps
    out = []
    for c in comps:
        S, Bv = c["vertices"], ind[c["kept"]]
        MSS = M[S][:, S].toarray()
        MSB = M[S][:, Bv].toarray()
        MBS = M[Bv][:, S].toarray()
        block = -(MBS @ np.linalg.solve(MSS, MSB)) if Bv.size else np.zeros((0, 0))
        out.append(dict(vertices=S, kept=c["kept"], block=block, kappa=float(np.linalg.cond(MSS))))
    return out


# Error bound of one block, per entry: C_BOUND * s * eps * kappa_2(M_SS) * max|block|.
# Entry (i, j) of either computation is y_i^T y_j with y = C^-1 M_SB.  The Cholesky factor (or the
# host's LU) is the exact factor of M_SS + dM with |dM| <= (s + 1) eps |C||C^T|, which moves the
# entry by at most ||y_i|| ||y_j|| ||dM|| / lambda_min <= (s + 1) eps kappa max|block| (to first
# order, ||y_i||^2 = |block_ii| <= max|block|); the forward substitution moves each y by s eps
# sqrt(kappa) ||y|| and the final dot product adds s eps ||y_i|| ||y_j||.  One side is at most
# 4 s eps kappa max|block|, and the kernel and the host reference each carry one.
C_BOUND = 8
EPS = float(np.finfo(np.float64).eps)


def block_bound(blk, c=C_BOUND):
    """Per-entry bound of one block of ``schur_blocks``."""
    if blk["block"].size == 0:
        return 0.0
    s = blk["vertices"].size
    return c * s * EPS * blk["kappa"] * float(np.abs(blk["block"]).max())


def schur_tolerance(M, ind, blocks, c=C_BOUND):
    """Per-entry tolerance (m x m) of the whole reduction M[ind, ind] + sum of the blocks: the
    bound of every block that touches the entry, plus k eps times the sum of the magnitudes of the
    entry's k terms for summing the blocks and M[ind, ind] (k - 1 roundings of at most eps / 2
    times that sum on each side)."""
    M = sparse.csr_matrix(M, dtype=np.float64)
    ind = np.asarray(ind, dtype=np.int64)
    m = ind.size
    mag = np.abs(M[ind][:, ind].toarray())
    terms = (mag != 0).astype(np.float64)
    tol = np.zeros((m, m))
    for blk in blocks:
        k = blk["kept"]
        if k.size:
            tol[np.ix_(k, k)] += block_bound(blk, c)
            mag[np.ix_(k, k)] += np.abs(blk["block"])
            terms[np.ix_(k, k)] += 1
    return tol + terms * EPS * mag


def sparsify_counts(k, q, seed):
    """Counts of gsp_sparsify_sample(k, q, seed), every draw replayed: draw d belongs to chunk
    d // 128 (Philox subsequence `chunk` of key `seed`) and is half of curand4 number
    t = (d - 128 chunk) // 2, words (x, y) for an even offset and (z, w) for an odd one, read as
    r = hi << 32 | lo; u = floor(r T / 2^64) with T the total weight, and the draw lands on the
    first edge e with cum[e] > u.  ``k``: the non-negative integer weights (total below 2^64)."""
    k = np.asarray(k, dtype=np.uint64)
    cum = np.cumsum(k, dtype=np.uint64)
    counts = np.zeros(k.size, dtype=np.int64)
    if q == 0 or k.size == 0:
        return counts
    T = int(cum[-1])
    d = np.arange(int(q), dtype=np.int64)
    chunk = d // DRAWS_PER_CHUNK
    off = d - chunk * DRAWS_PER_CHUNK
    x, y, z, w = curand4(int(seed), chunk.astype(np.uint64), (off // 2).astype(np.uint64))
    u32 = np.uint64(32)
    r = np.where(off % 2 == 0, (x << u32) | y, (z << u32) | w)
    u = ((r.astype(object) * T) >> 64).astype(np.uint64)
    e = np.searchsorted(cum, u, side="right")
    return np.bincount(e, minlength=k.size).astype(np.int64)
