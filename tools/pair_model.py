"""CPU model of the HBM traffic of two middle Clenshaw steps: two launches against one paired launch.

    python tools/pair_model.py [--graph config2|knn10m|config3] [--l2 24 32 40] [--rows 64]
                               [--nsig 64]

A middle Clenshaw step forms b_k = a2 L b_{k+1} - 2 b_{k+1} - b_{k+2} + c_k x on row tiles of
`--rows` rows.  Two schedules of two consecutive steps are replayed through ONE LRU cache of signal
rows (a row is nsig * 4 bytes) that stands in for the L2; its capacity under the streaming
operands is not known, so several sizes are reported.

  two launches  today: step k walks the tiles in one direction, step k-1 in the other; b_k is
                written over b_{k+2} (two blocks).
  paired        one launch of 2 T slots: A(t) forms b_k on tile t, B(t) forms b_{k-1}; the A tiles
                keep today's order and B(t) sits directly after the slot of the last A tile among
                t and the tiles its rows reference (pair_slots below).  Three blocks: A gathers P,
                reads Q, writes W; B gathers W, reads P, writes over Q.

What the replay counts is row fills from HBM.  A gather touches each distinct column of a tile
once (repeats inside a tile are L1's business, tools/gather_model.py).  Reads that are a block's
last use in the launch (evict-first loads) do not allocate: a hit frees the row, a miss is a
fill.  Full-row stores allocate without a fill.  Every written row goes back to HBM once in both
schedules (the next pair reads it), so write-backs are 2 N rows per pair either way, and the CSR
slabs (evict-first bulk copies) are 2 passes either way; both are added as constants.  Slots are
replayed one after the other: the 396 tiles that run at once on the device (6.5 MB per block at
64 signals) are not interleaved, so the model is an estimate, not a measurement.  The count is
taken on the second of two pairs (four steps), when the cache holds what the previous pair left.
DESIGN.md section 4.1 sets the table beside the measured times of cheby_pair_tiled, which places
B(t) a lag of A tiles later than this replay does (slots that are neighbours run at the same time)
and gains a quarter of the modelled bytes on config 2.
"""
import argparse
import os
import sys
import time
from collections import OrderedDict

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def tile_columns(indptr, indices, T, R):
    """Distinct columns of each of the T tiles of R rows."""
    return [np.unique(indices[indptr[t * R]:indptr[t * R + R]]) for t in range(T)]


def tile_neighbours(cols, T, R):
    """nbr[t]: the distinct tiles (< T) that the rows of tile t reference, t included."""
    out = []
    for t in range(T):
        nb = np.unique(cols[t] // R)
        nb = nb[nb < T]
        out.append(np.union1d(nb, [t]))
    return out


def pair_slots(nbr, T, reverse):
    """Slot table of one paired launch: a list of (tile, which), which = 0 for A, 1 for B.

    The A tiles come in walk order; B(t) is placed directly after the A tile that is last in
    walk order among nbr[t]."""
    pos = np.arange(T)[::-1] if reverse else np.arange(T)        # pos[t]: rank of A(t)
    last = np.array([pos[nb].max() for nb in nbr])               # rank after which B(t) may run
    order = np.argsort(pos, kind="stable")                       # tiles by A rank
    by_last = [[] for _ in range(T)]
    for t in (range(T - 1, -1, -1) if reverse else range(T)):
        by_last[last[t]].append(t)
    slots = []
    for rank in range(T):
        slots.append((int(order[rank]), 0))
        slots.extend((t, 1) for t in by_last[rank])
    return slots


class L2:
    def __init__(self, cap_rows):
        self.cap, self.d, self.fills = cap_rows, OrderedDict(), 0

    def touch(self, key):
        d = self.d
        if key in d:
            d.move_to_end(key)
            return
        self.fills += 1
        d[key] = None
        if len(d) > self.cap:
            d.popitem(last=False)

    def last_use(self, key):
        if self.d.pop(key, 0) == 0:
            self.fills += 1

    def write(self, key):
        d = self.d
        if key in d:
            d.move_to_end(key)
            return
        d[key] = None
        if len(d) > self.cap:
            d.popitem(last=False)


def run_tile(l2, n, R, cols, t, gathered, own_last, out, x_keep):
    """One tile of one step: gather block `gathered`, read own rows of `own_last` (last use) and
    of the source x (block 3; kept when x_keep), write own rows of `out`."""
    g = gathered * n
    for c in cols[t].tolist():
        l2.touch(g + c)
    r0 = t * R
    o, w, x = own_last * n + r0, out * n + r0, 3 * n + r0
    for r in range(R):
        l2.last_use(o + r)
        if x_keep:
            l2.touch(x + r)
        else:
            l2.last_use(x + r)
        l2.write(w + r)


def two_launches(n, R, T, cols, cap_rows):
    """Fills of steps 3 and 4 of four single steps (blocks 0 and 1, alternating direction)."""
    l2 = L2(cap_rows)
    cur, old = 0, 1
    for step in range(4):
        if step == 2:
            l2.fills = 0
        tiles = range(T - 1, -1, -1) if step & 1 else range(T)
        for t in tiles:
            run_tile(l2, n, R, cols, t, cur, old, old, False)
        cur, old = old, cur
    return l2.fills


def paired(n, R, T, cols, nbr, cap_rows):
    """Fills of the second of two paired launches (blocks 0, 1, 2 rotating), and its slots."""
    l2 = L2(cap_rows)
    P, Q, W = 0, 1, 2
    for pair in range(2):
        if pair == 1:
            l2.fills = 0
        slots = pair_slots(nbr, T, reverse=bool(pair & 1))
        for t, which in slots:
            if which == 0:
                run_tile(l2, n, R, cols, t, P, Q, W, True)
            else:
                run_tile(l2, n, R, cols, t, W, P, Q, False)
        P, Q, W = Q, W, P
    return l2.fills, slots


def main():
    import gather_model as gm
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--graph", default="config2", choices=["config2", "knn10m", "config3"])
    ap.add_argument("--l2", type=int, nargs="+", default=[24, 32, 40], help="LRU sizes in MB")
    ap.add_argument("--rows", type=int, default=64)
    ap.add_argument("--nsig", type=int, default=64)
    a = ap.parse_args()
    t0 = time.time()
    if a.graph == "config2":
        n, rows = gm.config2_rows()
    elif a.graph == "knn10m":
        n, rows = gm.config2_rows(10_000_000)
    else:
        n, rows = gm.grid_rows()
    R = a.rows
    T = n // R
    cols = tile_columns(rows.indptr, rows.indices, T, R)
    nbr = tile_neighbours(cols, T, R)
    nnz = int(rows.indptr[T * R])
    row_bytes = a.nsig * 4
    csr = 2 * (8 * nnz + 4 * n)                     # two steps' slabs
    writes = 2 * T * R * row_bytes
    print("graph %s: %d rows, %d tiles of %d, %.1f neighbour tiles per tile (max %d); %.0f s" % (
        a.graph, n, T, R, np.mean([len(b) for b in nbr]), max(len(b) for b in nbr),
        time.time() - t0), flush=True)
    slots = pair_slots(nbr, T, False)
    where = {}
    for i, s in enumerate(slots):
        where[s] = i
    late = np.array([where[(t, 1)] - where[(t, 0)] for t in range(T)])
    print("slot(B(t)) - slot(A(t)): median %d, 90%% %d, 99%% %d, max %d; beyond 2 x 396 slots: "
          "%.1f%%, beyond 2000: %.1f%%" % (np.median(late), np.percentile(late, 90),
                                          np.percentile(late, 99), late.max(),
                                          100 * (late > 792).mean(), 100 * (late > 2000).mean()))
    print("| L2 model | two launches, MB per pair | paired, MB per pair | paired / two |")
    print("|---|---|---|---|")
    for mb in a.l2:
        cap = mb * (1 << 20) // row_bytes
        f2 = two_launches(n, R, T, cols, cap) * row_bytes + csr + writes
        fp, _ = paired(n, R, T, cols, nbr, cap)
        fp = fp * row_bytes + csr + writes
        print("| %d MB | %.0f | %.0f | %.2f |" % (mb, f2 / 1e6, fp / 1e6, fp / f2), flush=True)
    print("(%.0f s)" % (time.time() - t0))


if __name__ == "__main__":
    main()
