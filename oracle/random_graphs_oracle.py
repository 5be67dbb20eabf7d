"""Serial restatements of the device random graph samplers (csrc/random_graphs.cu), and the
exact law of the reference's sequential Barabasi-Albert process for tiny graphs.

Test infrastructure: nothing under pygsp_b200/ imports this module.

* ``philox4x32_10`` -- Philox4x32-10 (Salmon et al., SC'11), as curand_kernel.h computes it.
  ``curand_init(key, subsequence, offset)`` with offset = 4 t followed by ``curand4`` returns
  ``philox4x32_10((t lo, t hi, subsequence lo, subsequence hi), (key lo, key hi))``, words in
  (x, y, z, w) order.
* ``sbm_graph`` -- the chunk plan, the decoders and the geometric-skip walk of gsp_sbm_count /
  gsp_sbm_fill; reproduces the device graph bit for bit.
* ``ba_graph`` -- the slot / attempt / rejection scheme of gsp_barabasi_albert, run slot by slot
  in order (every pointee is then already final); the device's rounds reach the same values.
* ``ba_exact_law`` -- probability of every labelled graph of barabasialbert.py:54-64 by
  enumeration, successive-sampling probabilities for choice(replace=False, p).
"""
import math

import numpy as np
from scipy import sparse

_M0, _M1 = 0xD2511F53, 0xCD9E8D57
_W0, _W1 = 0x9E3779B9, 0xBB67AE85
_MASK = 0xFFFFFFFF
RECT, TRI_STRICT, TRI_LOOPS, OFF_DIAG = 0, 1, 2, 3


def philox4x32_10(ctr, key):
    """Philox4x32-10 of counter words ctr = (c0, c1, c2, c3) and key words (k0, k1).  Words are
    Python ints or uint64 numpy arrays holding 32-bit values (element-wise)."""
    c0, c1, c2, c3 = ctr
    k0, k1 = key
    for r in range(10):
        if r:
            k0, k1 = (k0 + _W0) & _MASK, (k1 + _W1) & _MASK
        p0, p1 = _M0 * c0, _M1 * c2
        c0, c1, c2, c3 = ((p1 >> 32) ^ c1 ^ k0) & _MASK, p1 & _MASK, \
                         ((p0 >> 32) ^ c3 ^ k1) & _MASK, p0 & _MASK
    return c0, c1, c2, c3


def curand4(key, subsequence, t):
    """The t-th curand4 of curand_init(key, subsequence, 0): four 32-bit words."""
    u = np.uint64
    sub = np.asarray(subsequence, dtype=np.uint64)
    t = np.asarray(t, dtype=np.uint64)
    return philox4x32_10((t & u(_MASK), t >> u(32), sub & u(_MASK), sub >> u(32)),
                         (u(key & _MASK), u(key >> 32)))


# ------------------------------------------------------------------ SBM --------------------
def pair_space(na, nb, same, directed, self_loops):
    if not same:
        return RECT, na * nb, nb
    if directed:
        return (RECT, na * na, na) if self_loops else (OFF_DIAG, na * (na - 1), na)
    return (TRI_LOOPS, na * (na + 1) // 2, na) if self_loops else (TRI_STRICT, na * (na - 1) // 2, na)


def decode(kind, idx, width):
    """Block-local (i, j) of one candidate index (Python ints, exact)."""
    if kind == RECT:
        return idx // width, idx % width
    if kind == OFF_DIAG:
        i, j = idx // (width - 1), idx % (width - 1)
        return i, j + (j >= i)
    if kind == TRI_STRICT:
        i = math.isqrt(8 * idx + 1)
        i = (i + 1) // 2
        while i * (i - 1) // 2 > idx:
            i -= 1
        while (i + 1) * i // 2 <= idx:
            i += 1
        return i, idx - i * (i - 1) // 2
    i = (math.isqrt(8 * idx + 1) - 1) // 2
    return i, idx - i * (i + 1) // 2


def chunk_plan(sizes, M, directed, self_loops, target=64):
    """Block pairs with their chunking: list of dicts in chunk order (b <= a when undirected)."""
    k = len(sizes)
    start = [0]
    for s in sizes[:-1]:
        start.append(start[-1] + int(s))
    plan, cfirst = [], 0
    for a in range(k):
        for b in range(k if directed else a + 1):
            kind, n, width = pair_space(int(sizes[a]), int(sizes[b]), a == b, directed, self_loops)
            p = float(M[a][b])
            if n == 0 or p == 0:
                continue
            clen = min(max(math.ceil(target / p), 1), n)
            nch = -(-n // clen)
            plan.append(dict(a=a, b=b, n=n, clen=clen, cfirst=cfirst, nch=nch, row0=start[a],
                             col0=start[b], width=width, kind=kind, p=p,
                             lq=math.log1p(-p) if p < 1 else -math.inf))
            cfirst += nch
    return plan


def walk(blk, key):
    """Successful candidate indices of one block pair, every chunk's walk (vectorised over the
    block pair's chunks, each walking its own stream in order)."""
    n, clen, nch = blk["n"], blk["clen"], blk["nch"]
    if blk["p"] >= 1.0:
        return np.arange(n, dtype=np.int64)
    local = np.arange(nch, dtype=np.int64)
    chunk = blk["cfirst"] + local
    end = np.minimum(local * clen + clen, n)
    pos = local * clen - 1
    found = []
    t = 0
    active = np.ones(nch, dtype=bool)
    while active.any():
        w = curand4(key, chunk[active].astype(np.uint64), t // 2)
        hi, lo = (w[0], w[1]) if t % 2 == 0 else (w[2], w[3])
        r = (hi << np.uint64(32)) | lo
        u = ((r >> np.uint64(11)) + np.uint64(1)).astype(np.float64) * 2.0 ** -53
        skip = np.floor(np.log(u) / blk["lq"])
        p_act, e_act = pos[active], end[active]
        go = skip < (e_act - p_act - 1).astype(np.float64)
        nxt = p_act + 1 + np.where(go, skip, 0).astype(np.int64)
        found.append(nxt[go])
        pos[active] = np.where(go, nxt, p_act)
        idx = np.flatnonzero(active)
        active[idx[~go]] = False
        t += 1
    return np.sort(np.concatenate(found)) if found else np.zeros(0, dtype=np.int64)


def sbm_graph(N, k, z, M, directed, self_loops, key, target=64):
    """(adjacency as canonical scipy CSR, number of emitted COO entries) of the device SBM."""
    z = np.asarray(z, dtype=np.int64)
    perm = np.argsort(z, kind="stable")
    sizes = np.bincount(z, minlength=k)
    rows, cols = [], []
    for blk in chunk_plan(sizes, M, directed, self_loops, target):
        for idx in walk(blk, key).tolist():
            i, j = decode(blk["kind"], idx, blk["width"])
            u, v = int(perm[blk["row0"] + i]), int(perm[blk["col0"] + j])
            rows.append(u)
            cols.append(v)
            if not directed and u != v:
                rows.append(v)
                cols.append(u)
    W = sparse.coo_matrix((np.ones(len(rows)), (rows, cols)), shape=(N, N)).tocsr()
    W.sum_duplicates()
    return W, len(rows)


# ------------------------------------------------------------------ BA ---------------------
def ba_targets(N, m0, m, key):
    """Final target of every slot (i, s), slot id (i - m0) m + s, serially."""
    target = [-1] * (m * max(N - m0, 0))
    for i in range(m0, N):
        w = i + 2 * m * (i - m0)
        base = (i - m0) * m
        for s in range(m):
            k = 0
            while True:
                slot = base + s
                x, y, _, _ = philox4x32_10((k & _MASK, k >> 32, slot & _MASK, slot >> 32),
                                           (key & _MASK, key >> 32))
                r = (((x << 32) | y) * w) >> 64
                if r < i:
                    v = r
                else:
                    q = r - i
                    v = m0 + (q >> 1) // m if q % 2 == 0 else target[q >> 1]
                if v in target[base:base + s]:
                    k += 1
                    continue
                target[slot] = v
                break
    return target


def ba_graph(N, m0, m, key):
    """Adjacency (canonical scipy CSR, unit weights) of the device Barabasi-Albert graph."""
    t = np.array(ba_targets(N, m0, m, key), dtype=np.int64)
    i = m0 + np.arange(t.size) // max(m, 1)
    W = sparse.coo_matrix((np.ones(2 * t.size), (np.concatenate([i, t]), np.concatenate([t, i]))),
                          shape=(N, N)).tocsr()
    W.sum_duplicates()
    return W


def _subsets(w, m):
    """{frozenset S: probability} of m successive draws without replacement, P(j) ~ w[j]."""
    out = {}

    def rec(chosen, prob, left):
        if len(chosen) == m:
            key = frozenset(chosen)
            out[key] = out.get(key, 0.0) + prob
            return
        for j, wj in enumerate(w):
            if j not in chosen:
                rec(chosen + [j], prob * wj / left, left - wj)
    rec([], 1.0, float(sum(w)))
    return out


def ba_exact_law(N, m0, m):
    """{frozenset of edges (v, i), v < i: probability} of the reference's sequential process."""
    law = {frozenset(): 1.0}
    for i in range(m0, N):
        nxt = {}
        for edges, prob in law.items():
            deg = [0] * i
            for v, u in edges:
                deg[v] += 1
                deg[u] += 1
            for S, ps in _subsets([1 + d for d in deg], m).items():
                g = edges | {(v, i) for v in S}
                nxt[g] = nxt.get(g, 0.0) + prob * ps
        law = nxt
    return law


def edge_set(W):
    """frozenset of the edges (v, i), v < i, of a symmetric scipy adjacency."""
    coo = sparse.triu(W, k=1).tocoo()
    return frozenset(zip(coo.row.tolist(), coo.col.tolist()))
