"""Host restatements of tree multiresolution (pygsp_b200.reduction.tree_multiresolution).

``tree_multiresolution_levels``: the coarsening rules of DESIGN.md section 4.21 in NumPy, with the
depths and parents taken from ``scipy.sparse.csgraph.breadth_first_order``, an algorithm
independent of the device's.  ``euler_tour_depths``: a vectorised NumPy restatement of the device's
rooting (csrc/tree.cu): arcs in CSR order, twins, successors, Wyllie ranking, orientation and the
+-1 scan, so that the rule can be checked against BFS without a GPU.
"""
import numpy as np
from scipy import sparse
from scipy.sparse import csgraph

METHODS = ("unweighted", "sum", "resistance_distance")


def symmetric_support(W):
    """Canonical CSR of a symmetric adjacency without its diagonal (the tree's edges)."""
    W = sparse.csr_matrix(W)
    W = W.copy()
    W.sum_duplicates()
    W.setdiag(0)
    W.eliminate_zeros()
    W.sort_indices()
    return W


def _arcs(Ws):
    """(src, dst, weight as float64) of the off-diagonal entries of Ws, in CSR order."""
    Ws = sparse.csr_matrix(Ws)
    rows = np.repeat(np.arange(Ws.shape[0]), np.diff(Ws.indptr))
    off = rows != Ws.indices
    return rows[off], Ws.indices[off].astype(np.int64), Ws.data[off].astype(np.float64)


def bfs_depths(Ws, root):
    """(depth, parent, weight to parent) of every vertex of the tree Ws from root, by BFS."""
    n = Ws.shape[0]
    order, pred = csgraph.breadth_first_order(sparse.csr_matrix(Ws), root, directed=False,
                                              return_predecessors=True)
    if order.size != n:
        raise ValueError("Graph is not connected")
    # hop distances from the root (SciPy's BFS in C): the depths of a tree
    depth = csgraph.shortest_path(sparse.csr_matrix(Ws), directed=False, unweighted=True,
                                  indices=root).astype(np.int64)
    parent = pred.astype(np.int64)
    parent[root] = root
    src, dst, w = _arcs(Ws)
    wpar = np.zeros(n, dtype=np.float64)
    down = parent[dst] == src
    down &= dst != root
    wpar[dst[down]] = w[down]
    return depth, parent, wpar


def euler_tour_depths(Ws, root):
    """The device's rooting, restated: (depth, parent, weight to parent) from the Euler tour."""
    n = Ws.shape[0]
    depth = np.zeros(n, dtype=np.int64)
    parent = np.full(n, root, dtype=np.int64)
    wpar = np.zeros(n, dtype=np.float64)
    src, dst, w = _arcs(Ws)
    n_arcs = src.size
    if n_arcs != 2 * (n - 1):
        raise ValueError("not a tree")
    if n_arcs == 0:
        return depth, parent, wpar
    arc_ptr = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(np.bincount(src, minlength=n), out=arc_ptr[1:])
    # twin: arc (v -> u) in row v; rows are sorted, so key (row, col) orders the arcs
    key = src * n + dst
    twin = np.searchsorted(key, dst * n + src)
    assert np.array_equal(key[twin], dst * n + src)
    succ = twin + 1
    wrap = succ == arc_ptr[dst + 1]
    succ[wrap] = arc_ptr[dst[wrap]]
    nxt = np.where(succ == arc_ptr[root], -1, succ)
    rank = (nxt != -1).astype(np.int64)
    reach = 1
    while reach < n_arcs:                     # Wyllie: ceil(log2 n_arcs) rounds
        live = nxt != -1
        j = nxt[live]
        new_rank, new_nxt = rank.copy(), nxt.copy()
        new_rank[live] = rank[live] + rank[j]
        new_nxt[live] = nxt[j]
        rank, nxt = new_rank, new_nxt
        reach *= 2
    pos = n_arcs - 1 - rank
    down = pos < pos[twin]
    step = np.empty(n_arcs, dtype=np.int64)
    step[pos] = np.where(down, 1, -1)
    scan = np.cumsum(step)
    parent[dst[down]] = src[down]
    wpar[dst[down]] = w[down]
    depth[dst[down]] = scan[pos[down]]
    return depth, parent, wpar


def combine(method, wv, wp):
    """New edge weights in float64 from the weights to the parent and to the grandparent."""
    wv, wp = np.asarray(wv, dtype=np.float64), np.asarray(wp, dtype=np.float64)
    if method == "unweighted":
        return np.ones_like(wv)
    if method == "sum":
        return wv + wp
    if method == "resistance_distance":
        return 1.0 / (1.0 / wv + 1.0 / wp)
    raise ValueError("Unknown graph reduction method.")


def tree_multiresolution_levels(W, Nlevel, method, root, dtype=np.float64, coords=None):
    """The levels of the tree multiresolution of the symmetric adjacency W (SciPy / NumPy).

    Returns a list of Nlevel dicts with 'keep' (ascending int64, ids of the level above), 'W'
    (canonical CSR of dtype), 'root', 'orig_idx' and 'coords' (when given).
    """
    dtype = np.dtype(dtype)
    Ws = symmetric_support(sparse.csr_matrix(W).astype(dtype))
    depth, parent, wpar = bfs_depths(Ws, root)
    orig = np.arange(Ws.shape[0])
    levels = []
    for _ in range(Nlevel):
        keep = np.flatnonzero(depth % 2 == 0)
        n_new = keep.size
        new_id = np.full(depth.size, -1, dtype=np.int64)
        new_id[keep] = np.arange(n_new)
        v = keep[keep != root]
        p = parent[v]
        g = parent[p]
        c = combine(method, wpar[v], wpar[p]).astype(dtype)
        i, j = new_id[v], new_id[g]
        Wn = sparse.csr_matrix((np.concatenate([c, c]), (np.concatenate([i, j]),
                                                        np.concatenate([j, i]))),
                               shape=(n_new, n_new), dtype=dtype)
        Wn.sum_duplicates()
        Wn.eliminate_zeros()
        Wn.sort_indices()
        new_parent = np.arange(n_new, dtype=np.int64)
        new_parent[i] = j
        new_wpar = np.zeros(n_new, dtype=np.float64)
        new_wpar[i] = c.astype(np.float64)
        root = int(new_id[root])
        orig = orig[keep]
        level = {"keep": keep, "W": Wn, "root": root, "orig_idx": orig,
                 "depth": depth[keep] // 2, "parent": new_parent}
        if coords is not None:
            coords = np.asarray(coords)[keep]
            level["coords"] = coords
        levels.append(level)
        depth, parent, wpar = depth[keep] // 2, new_parent, new_wpar
    return levels


def random_tree(n, seed, relabel=True, decades=6):
    """A random recursive tree on n vertices (vertex k > 0 joins a uniform earlier vertex),
    randomly relabelled, with weights 10^U(0, decades): a symmetric SciPy CSR float64 matrix."""
    rng = np.random.default_rng(seed)
    if n == 1:
        return sparse.csr_matrix((1, 1), dtype=np.float64)
    child = np.arange(1, n)
    par = (rng.random(n - 1) * child).astype(np.int64)
    w = 10.0 ** (rng.random(n - 1) * decades)
    perm = rng.permutation(n) if relabel else np.arange(n)
    u, v = perm[child], perm[par]
    W = sparse.csr_matrix((np.concatenate([w, w]), (np.concatenate([u, v]), np.concatenate([v, u]))),
                          shape=(n, n))
    W.sort_indices()
    return W
