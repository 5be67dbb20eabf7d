"""The neighbour rings of the tiled Clenshaw steps (gsp_cheby_ring_plan_host), without a GPU.

The builder is host code, so the tables checked here are the ones the kernels read.  Against a
numpy construction, for every graph and tile size: the ring of each full tile is the sorted union
of its own rows and its columns, the runs cover it in order with maximal stretches of consecutive
rows, the ring position of the tile's first row, the largest ring, and ring[local[j]] == indices[j]
for every stored entry of a full tile.  Also: a tile whose ring is a single run, and the counts
alone when the run table has too little room.
"""
import ctypes

import numpy as np
import pytest

from pygsp_b200 import _native as nat

from test_clenshaw_pairs_cpu import GRAPHS


def ring_plan(L, R, cap=None):
    n, T = L.shape[0], L.shape[0] // R
    indptr = np.ascontiguousarray(L.indptr, dtype=np.int32)
    indices = np.ascontiguousarray(L.indices, dtype=np.int32)
    count, ring_max = ctypes.c_int64(0), ctypes.c_int32(0)
    cap = cap if cap is not None else L.nnz + T
    meta = np.full(4 * T, -1, np.int32)
    runs = np.full(2 * max(cap, 1), -1, np.int32)
    local = np.full(max(L.nnz, 1), 0xffff, np.uint16)
    nat.call("gsp_cheby_ring_plan_host", nat.i64(n), indptr, indices, nat.i32(R), nat.i64(cap),
             meta, runs, local, ctypes.byref(count), ctypes.byref(ring_max))
    return meta.reshape(T, 4), runs[:2 * count.value].reshape(-1, 2), local, count.value, ring_max.value


def _rings(L, R):
    T = L.shape[0] // R
    return [np.union1d(np.arange(t * R, t * R + R), L.indices[L.indptr[t * R]:L.indptr[t * R + R]])
            for t in range(T)]


@pytest.mark.parametrize("name", sorted(GRAPHS))
@pytest.mark.parametrize("R", [8, 32, 64])
def test_ring_plan_matches_numpy(name, R):
    L = GRAPHS[name]
    meta, runs, local, n_runs, ring_max = ring_plan(L, R)
    rings = _rings(L, R)
    assert ring_max == max(len(r) for r in rings)
    assert meta[0, 0] == 0 and meta[-1, 1] == n_runs == len(runs)
    for t, ring in enumerate(rings):
        first, end, size, self_pos = meta[t]
        assert size == len(ring) and ring[self_pos] == t * R
        if t + 1 < len(rings):
            assert meta[t + 1, 0] == end
        # the runs: maximal stretches of consecutive rows, in ring order
        starts = np.flatnonzero(np.diff(ring, prepend=-2) != 1)
        assert np.array_equal(runs[first:end, 0], ring[starts])
        assert np.array_equal(runs[first:end, 1], starts)
        j0, j1 = L.indptr[t * R], L.indptr[t * R + R]
        assert np.array_equal(ring[local[j0:j1].astype(np.int64)], L.indices[j0:j1])
    tail = local[L.indptr[len(rings) * R]:L.nnz]
    assert (tail == 0).all()                            # rows past the last full tile


def test_single_run_ring():
    """A path: every tile's ring is its own rows and one row on each side, one run."""
    meta, _, _, n_runs, ring_max = ring_plan(GRAPHS["path"], 32)
    assert (meta[:, 1] - meta[:, 0] == 1).all() and n_runs == len(meta)
    assert ring_max == 34 and meta[0, 2] == 33 and meta[-1, 2] == 34


def test_largest_ring_is_reported():
    """The star's centre row references every vertex: its tile's ring is the whole graph, the
    others stay small, and ring_max is exactly that ring."""
    L = GRAPHS["star"]
    meta, _, _, _, ring_max = ring_plan(L, 32)
    assert ring_max == L.shape[0] == meta[:, 2].max()
    assert np.sort(meta[:, 2])[-2] < 100


def test_counts_only_without_room():
    L = GRAPHS["morton k-NN"]
    full = ring_plan(L, 64)
    meta, runs, local, n_runs, ring_max = ring_plan(L, 64, cap=1)
    assert n_runs == full[3] and ring_max == full[4]
    assert (meta == -1).all() and (local == 0xffff).all()


def test_sensor_graph_rings_are_small():
    """A Morton-ordered k-NN graph: the rings are a small multiple of the tile."""
    L = GRAPHS["morton k-NN"]
    meta, _, _, _, ring_max = ring_plan(L, 64)
    assert meta[:, 2].mean() < 4 * 64 and ring_max < 8 * 64
