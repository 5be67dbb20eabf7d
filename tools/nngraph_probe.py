"""Timing of the exhaustive neighbour search (csrc/neighbors.cu) against scipy's cKDTree.

    python tools/nngraph_probe.py [--reps 5] [--host]

k-NN at (N, d, k) = (65536, 27, 10) -- the 3x3 patches of a 256 x 256 RGB image -- and at
(200000, 64, 10), plus one radius search, on seeded normal clouds.  Device times are CUDA-event
medians after one warm-up call.  The achieved FP64 rate uses the model of DESIGN.md 4.13:
3 d flops per (query, candidate) pair for p = 1 and 2 (difference, product / absolute value,
sum), N^2 3 d in all.  With --host the same searches run through cKDTree on the host's CPUs
(workers=-1) for comparison: the tree build plus the time of the first --host-queries queries
scaled to N (the full host search at N = 2e5, d = 64 takes about ten minutes).  Prints one JSON
line per case.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def timed(torch, fn, reps):
    fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        out.append(a.elapsed_time(b) * 1e-3)
    return float(np.median(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--host", action="store_true")
    ap.add_argument("--host-queries", type=int, default=4096)
    args = ap.parse_args()
    import torch
    from scipy import spatial

    from pygsp_b200.graphs import knn_device, radius_device
    props = torch.cuda.get_device_properties(0)
    cases = [("knn", 65536, 27, 10, 2.0), ("knn", 200000, 64, 10, 2.0),
             ("knn", 65536, 27, 10, 1.0), ("radius", 65536, 27, None, 2.0)]
    for kind, n, d, k, p in cases:
        X = np.random.default_rng(n + d).normal(size=(n, d))
        pts = torch.from_numpy(X).cuda()
        if kind == "knn":
            sec = timed(torch, lambda: knn_device(pts, k, p=p), args.reps)
            extra = {"k": k}
        else:
            nn, dist = knn_device(pts, 10, p=p)
            eps = float(dist[:, 4].median().item())         # about 5 neighbours per point
            sec = timed(torch, lambda: radius_device(pts, eps, p=p), args.reps)
            extra = {"epsilon": eps, "nnz": radius_device(pts, eps, p=p).nnz}
        flops = 3.0 * d * float(n) * float(n)
        row = {"case": kind, "n": n, "d": d, "p": p, "device_s": sec,
               "fp64_tflops": flops / sec / 1e12, "gpu": props.name, **extra}
        if args.host:      # queries of the first m points, scaled to n (tree build included)
            m = min(n, args.host_queries)
            t0 = time.perf_counter()
            tree = spatial.cKDTree(X)
            t1 = time.perf_counter()
            if kind == "knn":
                tree.query(X[:m], k=k + 1, p=p, workers=-1)
            else:
                tree.query_ball_point(X[:m], r=eps, p=p, workers=-1)
            t2 = time.perf_counter()
            row["host_ckdtree_s"] = (t1 - t0) + (t2 - t1) * n / m
            row["host_queries_timed"] = m
            row["host_cpus"] = len(os.sched_getaffinity(0))
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
