"""Serial restatement of the exact-size subset sampler (gsp_sbm_count / gsp_sbm_fill walked at
an inflated probability, then gsp_subset_select), and a direct-difference SwissRoll.

Test infrastructure: nothing under pygsp_b200/ imports this module.

* ``subset_pairs`` -- the plan, the walk (random_graphs_oracle.walk), the redraw of a short walk
  with the next key, the Philox priorities of the global pair index and the (priority,
  candidate) selection; reproduces the device's COO entries bit for bit.
* ``swissroll_weights`` -- exp(-d^2 / (2 s^2)) >= thresh over every pair from float64 direct
  differences, the brute-force reference of the device's SwissRoll.
* ``swissroll_reference`` -- the reference's own dense SwissRoll weights (Gram expansion), the
  operations of swissroll.py in its order; the fixture keeps only a digest of its weights.
"""
import math

import numpy as np
from scipy import sparse

from . import random_graphs_oracle as rgo

RECT, TRI_STRICT = rgo.RECT, rgo.TRI_STRICT
MISS_LOG = math.log(1e12)
KEY_STEP = 0x9E3779B97F4A7C15


def inflated_probability(n, M):
    if n <= 0:
        return 0.0
    d = MISS_LOG + math.sqrt(MISS_LOG * MISS_LOG + 2.0 * MISS_LOG * n)
    return 1.0 if n + d >= M else (n + d) / M


def _plan(spaces, target):
    """Per space: (blocks as random_graphs_oracle.walk dicts, n)."""
    out, cfirst = [], 0
    for blocks, n in spaces:
        M = sum(b[1] for b in blocks)
        p = inflated_probability(n, M)
        walked = []
        for kind, n_pairs, width, row0, col0 in blocks:
            if n == 0 or n_pairs == 0:
                continue
            clen = min(max(math.ceil(target / p), 1), n_pairs)
            nch = -(-n_pairs // clen)
            walked.append(dict(n=n_pairs, clen=clen, cfirst=cfirst, nch=nch, kind=kind,
                               width=width, row0=row0, col0=col0, p=p,
                               lq=math.log1p(-p) if p < 1 else -math.inf))
            cfirst += nch
        out.append((walked, n))
    return out


def priorities(key, u, v, N):
    """64-bit priority of the pairs (u, v): words x, y of the Philox block (u N + v, 2^63)."""
    g = np.asarray(u, dtype=np.uint64) * np.uint64(N) + np.asarray(v, dtype=np.uint64)
    w = rgo.curand4(key, np.uint64(1 << 63), g)
    return (w[0] << np.uint64(32)) | w[1]


def subset_pairs(N, spaces, key, target=64):
    """(rows, cols, attempt) int64: the device's 2 sum(n) COO entries, (u, v) then (v, u) per
    kept pair, space after space.  ``spaces`` as pygsp_b200.graphs.sampled.subset_plan."""
    plan = _plan(spaces, target)
    attempt = 0
    while True:
        wkey = (int(key) + attempt * KEY_STEP) % 2 ** 64
        cands = []
        for walked, n in plan:
            us, vs = [], []
            for blk in walked:
                idx = rgo.walk(blk, wkey)
                ij = [rgo.decode(blk["kind"], int(t), blk["width"]) for t in idx.tolist()]
                us += [blk["row0"] + i for i, _ in ij]
                vs += [blk["col0"] + j for _, j in ij]
            cands.append((np.array(us, dtype=np.int64), np.array(vs, dtype=np.int64), n))
        if all(u.size >= n for u, _, n in cands):
            break
        attempt += 1
    rows, cols = [], []
    for u, v, n in cands:
        if n == 0:
            continue
        prio = priorities(key, u, v, N)
        keep = np.lexsort((np.arange(u.size), prio))[:n]
        pair_rows = np.stack([u[keep], v[keep]], axis=1).ravel()
        pair_cols = np.stack([v[keep], u[keep]], axis=1).ravel()
        rows.append(pair_rows)
        cols.append(pair_cols)
    if not rows:
        return np.zeros(0, np.int64), np.zeros(0, np.int64), attempt
    return np.concatenate(rows), np.concatenate(cols), attempt


def swissroll_weights(coords, s, thresh):
    """Scipy CSR of W_ij = exp(-d_ij^2 / (2 s^2)), i != j, kept where W >= thresh and W > 0,
    d from float64 direct differences of the (N, dim) points."""
    X = np.asarray(coords, dtype=np.float64)
    n = X.shape[0]
    rows, cols, vals = [], [], []
    for i in range(n):
        diff = X - X[i]
        d2 = np.zeros(n)
        for k in range(X.shape[1]):
            d2 = d2 + diff[:, k] * diff[:, k]
        w = np.exp(-(np.sqrt(d2) ** 2) / (2.0 * s ** 2))
        keep = (w >= thresh) & (w > 0)
        keep[i] = False
        j = np.flatnonzero(keep)
        rows.append(np.full(j.size, i))
        cols.append(j)
        vals.append(w[j])
    return sparse.csr_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))),
                             shape=(n, n))


def swissroll_reference(coords, s, thresh):
    """Strict upper triangle (scipy CSR, sorted) of the reference's SwissRoll W from its
    coordinates (N, dim): swissroll.py's dense exp(-distanz(x)^2 / (2 s^2)) with the Gram
    expansion of utils.distanz, the diagonal removed and entries below thresh zeroed -- the
    same NumPy operations in the same order, so the same bits on the same NumPy."""
    x = np.asarray(coords, dtype=np.float64).T
    c = x.shape[1]
    xx = (x * x).sum(axis=0)
    xy = np.dot(x.T, x)
    dist = np.sqrt(abs(np.kron(np.ones((c, 1)), xx).T + np.kron(np.ones((c, 1)), xx) - 2 * xy))
    W = np.exp(-np.power(dist, 2) / (2.0 * s ** 2))
    W -= np.diag(np.diag(W))
    W[W < thresh] = 0
    T = sparse.triu(sparse.csr_matrix(W), k=1).tocsr()
    T.sort_indices()
    return T
