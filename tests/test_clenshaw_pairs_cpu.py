"""The slot table of the paired Clenshaw launch (csrc/pair_plan.cu), without a GPU.

The builder is host code, so the tables checked here are the ones the kernel walks.  For every
graph and lag: each tile appears once as step A and once as step B; B(t) follows A(s) for every
tile s that t's rows reference and for t itself, by at least the lag; a round-robin replay with
any number of CTAs, each taking its slots in order, never blocks; and replaying one pair tile by
tile in slot order on three blocks gives exactly what two plain steps give, which pins the block
rotation.
"""
import ctypes

import numpy as np
import pytest
from scipy import sparse

from oracle import step_oracle as so
from pygsp_b200 import _native as nat


def _laplacian(W):
    W = sparse.csr_matrix(W)
    L = (sparse.diags(np.asarray(W.sum(axis=1)).ravel()) - W).tocsr().astype(np.float32)
    L.sort_indices()
    return L


def _graphs():
    rng = np.random.default_rng(5)
    side = 40
    idx = np.arange(side * side).reshape(side, side)
    ends = np.concatenate([np.stack([idx[:, :-1].ravel(), idx[:, 1:].ravel()]),
                           np.stack([idx[:-1].ravel(), idx[1:].ravel()])], axis=1)
    grid = sparse.coo_matrix((np.ones(ends.shape[1]), (ends[0], ends[1])), shape=(idx.size,) * 2)
    knn = so.sensor_adjacency(3000, k=8, seed=3)
    path = sparse.diags([np.ones(999)], [1], shape=(1000, 1000))
    star = sparse.lil_matrix((1500, 1500))
    star[700, :] = 1.0
    star[700, 700] = 0.0
    star = sparse.csr_matrix(star)
    chain = sparse.diags([np.ones(1499)], [1], shape=(1500, 1500))
    p = rng.permutation(3000)
    one_way = sparse.triu(knn, 1).tocsr()          # a structure that is not symmetric
    return {"grid": _laplacian(grid + grid.T), "morton k-NN": _laplacian(knn),
            "path": _laplacian(path + path.T),
            "star": _laplacian(star + star.T + chain + chain.T),
            "permuted k-NN": _laplacian(knn[p][:, p]),
            "one-way": (one_way + sparse.identity(3000)).tocsr().astype(np.float32)}


GRAPHS = _graphs()


def pair_plan(L, R, lag):
    n, T = L.shape[0], L.shape[0] // R
    indptr = np.ascontiguousarray(L.indptr, dtype=np.int32)
    indices = np.ascontiguousarray(L.indices, dtype=np.int32)
    count = ctypes.c_int64(0)
    cap = 4
    for _ in range(2):
        nbr_ptr, nbr_idx = np.zeros(T + 1, np.int32), np.zeros(cap, np.int32)
        fwd, rev = np.full(2 * T, -1, np.int32), np.full(2 * T, -1, np.int32)
        nat.call("gsp_cheby_pair_plan_host", nat.i64(n), indptr, indices, nat.i32(R), nat.i32(lag),
                 nat.i64(cap), nbr_ptr, nbr_idx, fwd, rev, ctypes.byref(count))
        if count.value <= cap:
            break
        assert (fwd == -1).all()                       # too little room: nothing is written
        cap = count.value
    return nbr_ptr, nbr_idx[:count.value], fwd, rev


def _neighbours(L, R):
    T = L.shape[0] // R
    out = []
    for t in range(T):
        c = np.unique(L.indices[L.indptr[t * R]:L.indptr[t * R + R]] // R)
        out.append(np.union1d(c[c < T], [t]))
    return out


@pytest.mark.parametrize("name", sorted(GRAPHS))
@pytest.mark.parametrize("R,lag", [(8, 0), (8, 5), (64, 3), (64, 256)])
def test_tables_are_topological_orders(name, R, lag):
    L = GRAPHS[name]
    T = L.shape[0] // R
    nbr_ptr, nbr_idx, fwd, rev = pair_plan(L, R, lag)
    want = _neighbours(L, R)
    for t in range(T):
        assert np.array_equal(nbr_idx[nbr_ptr[t]:nbr_ptr[t + 1]], want[t])
    for slots, a_order in ((fwd, np.arange(T)), (rev, np.arange(T)[::-1])):
        tile, which = slots >> 1, slots & 1
        assert np.array_equal(tile[which == 0], a_order)
        assert np.array_equal(np.sort(tile[which == 1]), np.arange(T))
        pos_a = np.empty(T, np.int64)
        pos_b = np.empty(T, np.int64)
        pos_a[tile[which == 0]] = np.flatnonzero(which == 0)
        pos_b[tile[which == 1]] = np.flatnonzero(which == 1)
        a_before = np.cumsum(which == 0)                  # A slots up to and including a slot
        for t in range(T):
            last = pos_a[want[t]].max()
            assert last < pos_b[t]
            # exactly `lag` further A tiles run between the last A tile needed and B(t),
            # fewer only at the end of the table
            between = a_before[pos_b[t]] - a_before[last]
            assert between == lag or (between < lag and a_before[pos_b[t]] == T)


@pytest.mark.parametrize("name", ["morton k-NN", "star", "permuted k-NN"])
def test_round_robin_replay_never_blocks(name):
    L, R = GRAPHS[name], 8
    T = L.shape[0] // R
    want = _neighbours(L, R)
    for lag in (0, 4):
        for slots in pair_plan(L, R, lag)[2:]:
            for ctas in (1, 2, 3, 7, 132, 396, 2 * T):
                nxt = list(range(min(ctas, 2 * T)))          # next slot of each CTA
                done_a = np.zeros(T, bool)
                left = 2 * T
                while left:
                    progressed = False
                    for b in range(len(nxt)):
                        while nxt[b] < 2 * T:
                            t, w = slots[nxt[b]] >> 1, slots[nxt[b]] & 1
                            if w and not done_a[want[t]].all():
                                break
                            if not w:
                                done_a[t] = True
                            nxt[b] += ctas
                            left -= 1
                            progressed = True
                    assert progressed, (name, ctas)


@pytest.mark.parametrize("name", ["morton k-NN", "one-way"])
def test_slot_order_replay_equals_two_steps(name):
    L, R, nsig = GRAPHS[name][:1024, :1024].tocsr(), 64, 4
    n = L.shape[0]
    rng = np.random.default_rng(9)
    P, Q, x = (so.scaled_signals(rng, n, nsig) for _ in range(3))
    a, b, g, ck_a, ck_b = 0.37, -2.0, -1.0, 0.8, -0.3

    def step(cur, old, ck):        # a L cur + b cur + g old + ck x, in float64
        new = so.step_reference(L, cur, old, None, a, b, g, [], [], False)[0]
        return new + np.float32(ck) * x.astype(np.float64)

    bk = step(P, Q, ck_a).astype(np.float32)
    ref = step(bk, P, ck_b).astype(np.float32)
    for slots in pair_plan(L, R, 2)[2:]:
        W = np.full((n, nsig), np.nan, np.float32)
        Qw = Q.copy()
        for code in slots:
            rows = slice((code >> 1) * R, (code >> 1) * R + R)
            if code & 1:
                Qw[rows] = step(W, P, ck_b)[rows].astype(np.float32)
            else:
                W[rows] = step(P, Qw, ck_a)[rows].astype(np.float32)
        assert np.array_equal(W, bk) and np.array_equal(Qw, ref)
