"""Timing of tree multiresolution (needs a GPU).

    python tools/tree_probe.py [--reps 5] [--levels 3] [--out FILE]

One JSON line per measurement (also appended to --out when given):
  card : GPU name, power limit and SM clock limit (nvidia-smi), read in the same run;
  tree : for Path(10^7), LowStretchTree(11) (4^11 vertices) and a 10^7-vertex random recursive
         tree (relabelled, weights over six decades), float32, resistance_distance:
         root_ms   -- the rooting alone (checks, Euler tour, ranking, depths: reduction._tree_root);
         cc_ms     -- of which the connectivity check (gsp_cc_labels_* on the symmetric adjacency);
         coarsen_ms -- the first level's kernels alone (gsp_tree_keep, the read of the new size,
                      gsp_tree_coarsen_*), without the COO assembly and the Graph;
         level_ms  -- each of the first --levels coarsenings alone (keep, coarsen, COO assembly and
                      the level's Graph with its Laplacian: reduction._tree_level);
         total_ms  -- tree_multiresolution(G, --levels) as a user calls it;
         host_*_s  -- the NumPy oracle on the same tree, one run each: BFS rooting
                      (oracle.tree_oracle.bfs_depths) and all levels (tree_multiresolution_levels).
Device times are milliseconds, the median of --reps calls after one warm-up call, each call timed by
CUDA events around synchronised work.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def emit(rec, out):
    line = json.dumps(rec)
    print(line, flush=True)
    if out:
        with open(out, "a") as fh:
            fh.write(line + "\n")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def median_ms(fn, reps):
    import torch
    fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        times.append(s.elapsed_time(e))
    return round(statistics.median(times), 3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--levels", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("tree_probe needs a CUDA device")
    import pygsp_b200 as gsp
    from pygsp_b200 import _native as nat
    from oracle import tree_oracle as tro
    red = gsp.reduction
    emit({"card": card()}, a.out)

    cases = [("Path(1e7)", lambda: gsp.graphs.Path(10 ** 7, dtype=np.float32)),
             ("LowStretchTree(11)", lambda: gsp.graphs.LowStretchTree(11, dtype=np.float32)),
             ("random(1e7)", lambda: gsp.graphs.Graph(tro.random_tree(10 ** 7, 1),
                                                      dtype=np.float32))]
    method = "resistance_distance"
    for name, build in cases:
        G = build()
        root = int(getattr(G, "root", 1))
        root_ms = median_ms(lambda: red._tree_root(G, root), a.reps)
        Ws_dev, n, st = G._symmetric_adjacency(), G.N, nat.stream_ptr(G.device)
        labels = torch.empty(n, dtype=torch.int32, device=G.device)
        ncomp = torch.empty(1, dtype=torch.int64, device=G.device)
        cc_ms = median_ms(lambda: nat.call("gsp_cc_labels_f32", nat.i64(n), Ws_dev.indptr,
                                           Ws_dev.indices, Ws_dev.data, nat.i32(0), labels, ncomp,
                                           st), a.reps)
        depth, parent, wpar = red._tree_root(G, root)

        def coarsen():
            new_id = torch.empty(n + 1, dtype=torch.int32, device=G.device)
            nat.call("gsp_tree_keep", nat.i64(n), depth, new_id, ncomp, st)
            m = int(ncomp.item())
            out = [torch.empty(k, dtype=t, device=G.device) for k, t in
                   ((m, torch.int64), (2 * m - 2, torch.int32), (2 * m - 2, torch.int32),
                    (2 * m - 2, torch.float32), (m, torch.int32), (m, torch.int32),
                    (m, torch.float64))]
            nat.call("gsp_tree_coarsen_f32", nat.i64(n), nat.i64(m), depth, parent, wpar, new_id,
                     nat.i32(root), nat.i32(2), *out, st)
        coarsen_ms = median_ms(coarsen, a.reps)
        level_ms, sizes, H, state = [], [G.N], G, red._tree_root(G, root) + (root,)
        for _ in range(a.levels):
            depth, parent, wpar, r = state
            level_ms.append(median_ms(lambda: red._tree_level(H, depth, parent, wpar, r, method),
                                      a.reps))
            _, H, r2, d2, p2, w2 = red._tree_level(H, depth, parent, wpar, r, method)
            state = (d2, p2, w2, r2)
            sizes.append(H.N)
        total_ms = median_ms(lambda: red.tree_multiresolution(G, a.levels, method), a.reps)
        Ws = G._symmetric_adjacency().to_scipy()
        t0 = time.perf_counter()
        tro.bfs_depths(tro.symmetric_support(Ws), root)
        t1 = time.perf_counter()
        tro.tree_multiresolution_levels(Ws, a.levels, method, root, dtype=np.float32)
        t2 = time.perf_counter()
        emit({"tree": name, "N": G.N, "levels": a.levels, "sizes": sizes,
              "root_ms": root_ms, "cc_ms": cc_ms,
              "coarsen_ms": coarsen_ms, "level_ms": level_ms, "total_ms": total_ms,
              "host_root_s": round(t1 - t0, 3), "host_all_levels_s": round(t2 - t1, 3)}, a.out)
        del G, H, state
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
