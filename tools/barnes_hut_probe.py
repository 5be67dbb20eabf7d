"""Timing and accuracy of the Barnes-Hut spring repulsion (csrc/barnes_hut.cu) against the exact
all-pairs one (csrc/layout.cu).

    python tools/barnes_hut_probe.py [--iters 5] [--sizes 10000,100000,1000000,10000000]

On Sensor(N, k=10, seed=0) in 2-D from a seeded uniform start, for theta in {0.5, 1.0}: the
median per-iteration time of ``gsp_spring_step_bh_*`` (CUDA events, after a warm-up of every
shape), the time of ``gsp_spring_bh_tree`` alone (bounding box, keys, sort, radix tree and
aggregation), and their difference (the walk and the update).  The exact step is timed at
N <= 1e6 in the same run.  From the NumPy oracle's walk (oracle/barnes_hut_oracle.py) of a
256-row sample: the mean cells and leaves visited per query, and the ratio of the per-row bound
(frontier Taylor term plus centroid rounding, as ``bh_step_bound`` uses it) to the force's norm
(median and largest).  The card's name and power limit come first.
One JSON line per case.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from layout_probe import card  # noqa: E402


def _time(fn, iters):
    import torch
    fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b) * 1e-3)
    return float(np.median(times)), float(min(times))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--sizes", default="10000,100000,1000000,10000000")
    ap.add_argument("--exact-max", type=int, default=1000000)
    args = ap.parse_args()
    import torch

    import pygsp_b200 as gsp
    from oracle import barnes_hut_oracle as bo
    from pygsp_b200 import _native as nat
    if not torch.cuda.is_available():
        raise SystemExit("barnes_hut_probe: no CUDA device")
    print(json.dumps({"case": "card", **card()}), flush=True)
    for n in [int(s) for s in args.sizes.split(",")]:
        G = gsp.graphs.Sensor(n, k=10, seed=0)
        W = G.W
        start = np.random.default_rng(0).uniform(size=(n, 2))
        cur = torch.as_tensor(start, device=G.device)
        nxt = torch.empty_like(cur)
        k = float(np.sqrt(1.0 / n))
        ids = torch.empty(n, dtype=torch.int32, device=G.device)
        children = torch.empty(2 * (n - 1), dtype=torch.int32, device=G.device)
        counts = torch.empty(n - 1, dtype=torch.int32, device=G.device)
        boxes = torch.empty(4 * (n - 1), dtype=torch.float64, device=G.device)
        cents = torch.empty(2 * (n - 1), dtype=torch.float64, device=G.device)

        def tree():
            nat.call("gsp_spring_bh_tree", nat.i64(n), nat.i32(2), cur, ids, children, counts,
                     boxes, cents, nat.stream_ptr(G.device))

        def bh(theta):
            return lambda: G._call("gsp_spring_step_bh", nat.i64(n), nat.i32(2), W.indptr,
                                   W.indices, W.data, nat.f64(k), nat.f64(0.1), None, cur, nxt,
                                   nat.f64(theta))

        def exact():
            G._call("gsp_spring_step", nat.i64(n), nat.i32(2), W.indptr, W.indices, W.data,
                    nat.f64(k), nat.f64(0.1), None, cur, nxt)
        # warm every shape first, then time them in the same call
        tree()
        for theta in (0.5, 1.0):
            bh(theta)()
        if n <= args.exact_max:
            exact()
        torch.cuda.synchronize()
        tree_s, _ = _time(tree, args.iters)
        exact_s = None
        if n <= args.exact_max:
            exact_s, _ = _time(exact, max(2, args.iters // 2))
        host_tree = bo.build_tree(start)
        rows = np.sort(np.random.default_rng(1).choice(n, 256, replace=False))
        for theta in (0.5, 1.0):
            step_s, step_min = _time(bh(theta), args.iters)
            w = bo.walk(host_tree, start[rows], theta)
            # the whole per-row bound bh_step_bound uses: Taylor frontier plus centroid rounding
            ratio = (w["bound"] + w["centroid"]) / np.sqrt((w["force"] ** 2).sum(axis=1))
            row = {"case": "sensor", "n": n, "dim": 2, "theta": theta,
                   "bh_iteration_s": step_s, "bh_iteration_s_min": step_min,
                   "tree_s": tree_s, "walk_and_update_s": step_s - tree_s,
                   "exact_iteration_s": exact_s,
                   "speedup": None if exact_s is None else exact_s / step_s,
                   "cells_per_query": float(w["cells"].mean()),
                   "leaves_per_query": float(w["leaves"].mean()),
                   "tree_height": int(host_tree["height"]),
                   "bound_over_force_median": float(np.median(ratio)),
                   "bound_over_force_max": float(ratio.max())}
            print(json.dumps(row), flush=True)
        del G, cur, nxt, ids, children, counts, boxes, cents, host_tree
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
