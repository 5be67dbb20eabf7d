"""Serial restatement of the device random regular sampler (csrc/random_regular.cu), and the exact
law of the reference's sequential stub pairing for tiny graphs.

Test infrastructure: nothing under pygsp_b200/ imports this module.

* ``random_regular_edges`` -- one degree-k graph as the device builds it: attempts, bulk pairing
  rounds (stable sort by Philox priority, pairs (2i, 2i+1), legality against the graph at the start
  of the round, the lower pair index winning a repeated edge, stable compaction of the rejected
  stubs), the sequential tail with its exact stuck check and draw cap, restarts, and the
  last attempt's switches.  The edge list comes out in the device's order.
* ``random_regular_graph`` -- the whole model: the complement for k > (N - 1) / 2, and the
  adjacency as canonical SciPy CSR; reproduces the device graph bit for bit.
* ``exact_law`` -- probability of every class of k-regular graph under the reference's rule
  (draw a uniform legal pair of stubs, add it; restart on a stuck pool), conditioned on success.
"""
import itertools

import numpy as np
from scipy import sparse

from . import random_graphs_oracle as rgo

# The determinism constants of include/gspb200.h (GSPB200_RR_*).
TAIL_STUBS = 4096
CHECK_AFTER = 32
TAIL_DRAWS = 1 << 22
SWITCH_DRAWS = 1 << 16
MAX_ROUNDS = 4096
TAIL_STREAM = 0xFFFFFFFF
SWITCH_STREAM = 0xFFFFFFFE


class _Stream:
    """curand4 blocks t = 0, 1, ... of one Philox subsequence, fetched in vectorised batches."""

    def __init__(self, key, sub, batch=256):
        self.key, self.sub, self.batch = key, sub, batch
        self.base, self.words = 0, []

    def __call__(self, t):
        if not self.base <= t < self.base + len(self.words):
            self.base = t
            w = rgo.curand4(self.key, np.uint64(self.sub),
                            np.arange(t, t + self.batch, dtype=np.uint64))
            self.words = list(zip(*(a.tolist() for a in w)))
        return self.words[t - self.base]


def _canon(u, v):
    return (min(u, v) << 32) | max(u, v)


def _mulhi(x, y, n):
    return (((x << 32) | y) * n) >> 64


def _any_legal(pool, present):
    vs = sorted(set(pool))
    return any(_canon(u, v) not in present for u, v in itertools.combinations(vs, 2))


def _round(pool, key, sub, present_keys):
    """One bulk round: (accepted (u, v) arrays in pair order, the new pool)."""
    w = rgo.curand4(key, np.uint64(sub), np.arange(pool.size, dtype=np.uint64))
    prio = (w[0] << np.uint64(32)) | w[1]
    s = pool[np.argsort(prio, kind="stable")]
    u, v = s[0::2], s[1::2]
    ck = (np.minimum(u, v) << 32) | np.maximum(u, v)
    legal = (u != v) & ~np.isin(ck, present_keys)
    idx = np.flatnonzero(legal)
    _, first = np.unique(ck[idx], return_index=True)
    acc = np.zeros(u.size, dtype=bool)
    acc[idx[first]] = True
    return u[acc], v[acc], np.stack([u[~acc], v[~acc]], axis=1).ravel()


def random_regular_edges(N, k, max_iter, key):
    """Edge list of the device sampler for degree k (no complement): (eu, ev, attempts, rounds,
    complete).  eu / ev are lists in the device's order; complete is False when the last
    attempt's switches ran out of draws and the partial graph was kept."""
    if N * k == 0:
        return [], [], 0, 0, True
    rounds = 0
    for a in range(max_iter):
        last = a == max_iter - 1
        pool = np.tile(np.arange(N, dtype=np.int64), k)
        eu, ev = [], []
        keys = np.zeros(0, dtype=np.int64)
        r = 0
        while pool.size > TAIL_STUBS:
            if r == MAX_ROUNDS:
                raise RuntimeError("the rounds did not finish")
            u, v, pool = _round(pool, key, (a << 32) | r, keys)
            eu += u.tolist()
            ev += v.tolist()
            keys = np.concatenate([keys, (np.minimum(u, v) << 32) | np.maximum(u, v)])
            r += 1
        rounds += r
        present = set(keys.tolist())
        pool, P = pool.tolist(), pool.size
        draw = _Stream(key, (a << 32) | TAIL_STREAM)
        t = 0
        while True:
            rej = 0
            while P > 0 and rej < CHECK_AFTER and t < TAIL_DRAWS:
                x, y, z, w = draw(t)
                t += 1
                i1, i2 = _mulhi(x, y, P), _mulhi(z, w, P)
                v1, v2 = pool[i1], pool[i2]
                if v1 != v2 and _canon(v1, v2) not in present:
                    present.add(_canon(v1, v2))
                    eu.append(v1)
                    ev.append(v2)
                    pool[max(i1, i2)] = pool[P - 1]
                    P -= 1
                    pool[min(i1, i2)] = pool[P - 1]
                    P -= 1
                    rej = 0
                else:
                    rej += 1
            if P == 0 or t >= TAIL_DRAWS or not _any_legal(pool[:P], present):
                break
        if P == 0:
            return eu, ev, a + 1, rounds, True
        if not last:
            continue
        switch = _Stream(key, (a << 32) | SWITCH_STREAM)
        t, E = 0, len(eu)
        for p in range(0, P, 2):
            sa, sb = pool[p], pool[p + 1]
            placed = False
            for _ in range(SWITCH_DRAWS):
                if E == 0:
                    break
                x, y, z, _w = switch(t)
                t += 1
                e = _mulhi(x, y, E)
                xv, yv = (ev[e], eu[e]) if z & 1 else (eu[e], ev[e])
                if xv in (sa, sb) or yv in (sa, sb):
                    continue
                if _canon(sa, xv) in present or _canon(sb, yv) in present:
                    continue
                present.discard(_canon(xv, yv))
                present.add(_canon(sa, xv))
                present.add(_canon(sb, yv))
                eu[e], ev[e] = sa, xv
                eu.append(sb)
                ev.append(yv)
                E += 1
                placed = True
                break
            if not placed:
                return eu, ev, a + 1, rounds, False
        return eu, ev, a + 1, rounds, True
    raise ValueError("max_iter must be at least 1")


def random_regular_graph(N, k, max_iter, key):
    """(adjacency as canonical scipy CSR, attempts, rounds) of the device RandomRegular."""
    kk = N - 1 - k if 2 * k > N - 1 else k
    eu, ev, attempts, rounds, _ = random_regular_edges(N, kk, max_iter, key)
    rows, cols = np.array(eu + ev, dtype=np.int64), np.array(ev + eu, dtype=np.int64)
    W = sparse.coo_matrix((np.ones(rows.size), (rows, cols)), shape=(N, N)).tocsr()
    W.sum_duplicates()
    if kk != k:
        C = np.ones((N, N)) - np.eye(N) - W.toarray()
        W = sparse.csr_matrix(C)
        W.sum_duplicates()
    return W, attempts, rounds


# ------------------------------------------------------------ exact law of the reference's rule ---
def regular_graphs(N, k):
    """Every labelled simple k-regular graph on N vertices, as tuples of edges (u, v), u < v."""
    out = []

    def rec(u, rem, edges):
        if u == N:
            out.append(tuple(edges))
            return
        if rem[u] == 0:
            rec(u + 1, rem, edges)
            return
        cand = [v for v in range(u + 1, N) if rem[v] > 0]
        for S in itertools.combinations(cand, rem[u]):
            r = rem[u]
            rem[u] = 0
            for v in S:
                rem[v] -= 1
            rec(u + 1, rem, edges + [(u, v) for v in S])
            for v in S:
                rem[v] += 1
            rem[u] = r
    rec(0, [k] * N, [])
    return out


def sequential_probability(N, k, edges):
    """Probability that one attempt of the sequential rule ends with exactly ``edges``: the sum over
    the orders of the edges of the product of r_u r_v / L, r the free stubs per vertex and L the
    number of legal stub pairs, by dynamic programming over subsets."""
    m = len(edges)
    f = np.zeros(1 << m)
    f[0] = 1.0
    for mask in range(1, 1 << m):
        for e in range(m):
            if not mask >> e & 1:
                continue
            prev = mask ^ (1 << e)
            if f[prev] == 0:
                continue
            r = [k] * N
            for b in range(m):
                if prev >> b & 1:
                    r[edges[b][0]] -= 1
                    r[edges[b][1]] -= 1
            R = sum(r)
            L = (R * R - sum(x * x for x in r)) // 2
            L -= sum(r[edges[b][0]] * r[edges[b][1]] for b in range(m) if prev >> b & 1)
            a, c = edges[e]
            f[mask] += f[prev] * r[a] * r[c] / L
    return f[-1]


def graph_class(N, edges):
    """Class of a graph: its adjacency spectrum rounded to 1e-6 (isomorphic graphs share it)."""
    A = np.zeros((N, N))
    for u, v in edges:
        A[u, v] = A[v, u] = 1
    return tuple(np.round(np.linalg.eigvalsh(A), 6) + 0.0)


def exact_law(N, k):
    """{class: probability} of the reference's rule conditioned on success.  The rule is exchangeable,
    so every labelled graph of one isomorphism class has the same probability; each class's is
    computed on two of its members, which must agree (a check that the spectrum separates the
    classes that occur here)."""
    members = {}
    for g in regular_graphs(N, k):
        members.setdefault(graph_class(N, g), []).append(g)
    law = {}
    for c, gs in members.items():
        p = [sequential_probability(N, k, g) for g in gs[:2]]
        if abs(p[0] - p[-1]) > 1e-12 * p[0]:
            raise AssertionError("class %r mixes graphs of different probability" % (c,))
        law[c] = p[0] * len(gs)
    total = sum(law.values())
    return {c: p / total for c, p in law.items()}
