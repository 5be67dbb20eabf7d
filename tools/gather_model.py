"""CPU model of the x_cur gather of the tiled Chebyshev step: L2 row fetches per row owned.

    python tools/gather_model.py [--graph config2|knn10m|config3] [--cap 760 600] [--every 13]
                                 [--sms 132]

Every stored entry of a row makes its CTA gather one x_cur row (256 B at 64 signals).  The model
keeps one LRU cache of x_cur rows per SM (`--cap` rows: 760 rows = 190 KB, the L1 left beside
the shared-memory stage rings of three CTAs) and counts the rows that miss it, i.e. the gathers
that go to L2, per row the SM owns (the compulsory figure is 1.0).  CTA b runs on SM b mod SMs;
an SM's CTAs are interleaved tile by tile, the rows of a tile are visited in order, and the
entries of a row in stored order.  Every `--every`-th SM is simulated.

Schedules (T tiles of R rows, grid = SMs x CTAs per SM):
  round-robin  CTA b runs tiles b, b + grid, ...            (cheby_step_tiled, csrc/cheby_tiled.cu)
  contiguous   CTA b runs [floor(b T / grid), floor((b + 1) T / grid))
  sm-run       one contiguous run per SM, its CTAs take successive tiles of it
  chunks-C     round-robin chunks of C consecutive tiles

Graphs: config2 is bench.host_graph(1e6, 10, 0) (cKDTree, Morton order); knn10m is the same
generator at 1e7 vertices, of which only the rows of the simulated SMs are built (forward and
reverse k-NN edges: exactly the rows of the symmetrised graph); config3 is the 3162 x 3162 grid
(row-major, 4-neighbour stencil).  Nothing here runs on a GPU: it is an estimate, an LRU at row
granularity, not the real L1.  DESIGN.md section 4.1 sets its numbers beside measured step times:
fewer modelled L2 fetches did not make the 1e6-vertex step faster.
"""
import argparse
import os
import sys
import time
from collections import OrderedDict

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


class Rows:
    """Column indices (with the diagonal: a Laplacian's pattern) of the rows the model visits."""

    def __init__(self, indptr, indices):
        self.indptr, self.indices = indptr, indices


def config2_rows(n=1_000_000, k=10, seed=0):
    import bench
    W = bench.host_graph(n, k, seed)
    L = (W + __import__("scipy").sparse.identity(n, format="csr")).tocsr()   # pattern of L
    L.sort_indices()
    return n, Rows(L.indptr, L.indices)


def knn_sample_rows(n, k, seed, wanted):
    """Rows `wanted` (bool mask) of the symmetrised k-NN pattern of bench.host_graph(n, k, seed),
    plus the diagonal, without building the other rows."""
    from scipy import spatial
    from pygsp_b200.graphs import morton_order
    coords = np.random.default_rng(seed).uniform(0, 1, (n, 2))
    coords = coords[morton_order(coords)]
    _, NN = spatial.cKDTree(coords).query(coords, k=k + 1, workers=-1)
    NN = NN[:, 1:]
    src = np.repeat(np.arange(n), k)
    dst = NN.ravel()
    fwd = wanted[src]                    # row i lists its own neighbours ...
    rev = wanted[dst]                    # ... and every j that lists i
    rows = np.concatenate([src[fwd], dst[rev], np.flatnonzero(wanted)])
    cols = np.concatenate([dst[fwd], src[rev], np.flatnonzero(wanted)])
    order = np.lexsort((cols, rows))
    rows, cols = rows[order], cols[order]
    keep = np.ones(rows.size, dtype=bool)
    keep[1:] = (rows[1:] != rows[:-1]) | (cols[1:] != cols[:-1])
    rows, cols = rows[keep], cols[keep]
    indptr = np.zeros(n + 1, dtype=np.int64)
    np.add.at(indptr, rows + 1, 1)
    return Rows(np.cumsum(indptr), cols)


def grid_rows(side=3162):
    n = side * side
    r = np.arange(n)
    x = r % side
    nb = [np.where(r >= side, r - side, -1), np.where(x > 0, r - 1, -1), r,
          np.where(x < side - 1, r + 1, -1), np.where(r < n - side, r + side, -1)]
    nb = np.stack(nb, axis=1)
    mask = nb >= 0
    indptr = np.concatenate([[0], np.cumsum(mask.sum(axis=1))])
    return n, Rows(indptr, nb[mask])


def schedule(name, T, grid):
    """Tile sequence of CTA b under a schedule: a function b -> sequence of tiles."""
    if name == "round-robin":
        return lambda b: range(b, T, grid)
    if name == "contiguous":
        return lambda b: range(b * T // grid, (b + 1) * T // grid)
    if name.startswith("chunks-"):
        C = int(name.split("-")[1])
        nch = -(-T // C)
        return lambda b: [t for ch in range(b, nch, grid) for t in range(ch * C, min(T, ch * C + C))]
    raise ValueError(name)


def sm_tiles(name, T, sms, cps, s):
    """Tile sequences of the CTAs of SM s."""
    if name == "sm-run":
        run = list(range(s * T // sms, (s + 1) * T // sms))
        return [run[j::cps] for j in range(cps)]
    f = schedule(name, T, sms * cps)
    return [list(f(s + j * sms)) for j in range(cps)]


def simulate(rows, seqs, R, cap):
    """(L2 row fetches, rows owned) of one SM running the CTAs' tile sequences `seqs`."""
    lru = OrderedDict()
    miss = owned = 0
    ip, ix = rows.indptr, rows.indices
    for i in range(max((len(s) for s in seqs), default=0)):
        for s in seqs:
            if i >= len(s):
                continue
            t = s[i]
            for r in range(t * R, t * R + R):
                owned += 1
                for c in ix[ip[r]:ip[r + 1]].tolist():
                    if c in lru:
                        lru.move_to_end(c)
                    else:
                        miss += 1
                        lru[c] = None
                        if len(lru) > cap:
                            lru.popitem(last=False)
    return miss, owned


def fetches_per_row(rows, n, name, R, cps, cap, sms, sample):
    T = n // R
    miss = owned = 0
    for s in sample:
        m, o = simulate(rows, sm_tiles(name, T, sms, cps, s), R, cap)
        miss += m
        owned += o
    return miss / max(owned, 1)


# (label, schedule, R, CTAs per SM): the table of DESIGN.md section 4.1
CASES = [("R = 64, 3 CTAs/SM, round-robin", "round-robin", 64, 3),
         ("R = 64, 3 CTAs/SM, contiguous runs", "contiguous", 64, 3),
         ("R = 64, 2 CTAs/SM, contiguous runs", "contiguous", 64, 2),
         ("R = 192, 1 CTA/SM, contiguous runs", "contiguous", 192, 1),
         ("R = 128, 1 CTA/SM, contiguous runs", "contiguous", 128, 1),
         ("R = 64, 3 CTAs/SM sharing one run per SM", "sm-run", 64, 3),
         ("R = 64, 3 CTAs/SM, round-robin chunks of 8", "chunks-8", 64, 3),
         ("R = 64, 3 CTAs/SM, round-robin chunks of 16", "chunks-16", 64, 3)]


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--graph", default="config2", choices=["config2", "knn10m", "config3"])
    ap.add_argument("--cap", type=int, nargs="+", default=[760, 600],
                    help="LRU capacity in x_cur rows per SM (760 rows = 190 KB at 64 signals)")
    ap.add_argument("--sms", type=int, default=132)
    ap.add_argument("--every", type=int, default=None,
                    help="simulate every N-th SM (default 13; 44 for the 1e7-row graphs)")
    a = ap.parse_args()
    every = a.every or (13 if a.graph == "config2" else 44)
    sample = list(range(0, a.sms, every))
    t0 = time.time()
    if a.graph == "config2":
        n, rows = config2_rows()
    elif a.graph == "config3":
        n, rows = grid_rows()
    else:
        n = 10_000_000
        wanted = np.zeros(n, dtype=bool)
        for _, name, R, cps in CASES:              # every row a simulated SM owns in any case
            T = n // R
            for s in sample:
                for seq in sm_tiles(name, T, a.sms, cps, s):
                    for t in seq:
                        wanted[t * R:(t + 1) * R] = True
        rows = knn_sample_rows(n, 10, 0, wanted)
    print("graph %s: %d rows, built in %.0f s; SMs simulated: %s" % (
        a.graph, n, time.time() - t0, sample), flush=True)
    if a.graph == "config2":
        ip, ix = rows.indptr, rows.indices
        own = np.repeat(np.arange(n), np.diff(ip))
        gap = np.abs(ix - own)
        print("entries per row %.2f; |col - row| <= 32: %.0f%%, <= 256: %.0f%%" % (
            ix.size / n, 100 * (gap <= 32).mean(), 100 * (gap <= 256).mean()))
        u = [np.unique(ix[ip[t * 64]:ip[t * 64 + 64]]).size for t in range(0, n // 64, 7)]
        print("distinct columns of a 64-row tile: %.2f x 64" % (np.mean(u) / 64))
    print("| schedule | " + " | ".join("%d rows" % c for c in a.cap) + " |")
    print("|---|" + "---|" * len(a.cap))
    for label, name, R, cps in CASES:
        vals = [fetches_per_row(rows, n, name, R, cps, c, a.sms, sample) for c in a.cap]
        print("| %s | %s |" % (label, " | ".join("%.2f" % v for v in vals)), flush=True)
    print("(L2 row fetches of the gather per row owned; %.0f s)" % (time.time() - t0))


if __name__ == "__main__":
    main()
