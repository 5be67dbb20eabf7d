"""Times the random graph models on the device (DESIGN.md section 4.16).

    python tools/random_graph_probe.py [--reps 3] [--skip-host]

* the config-4 SBM of bench.py (N = 1e7, k = 8, p = 5e-6, q = 5e-7) sampled on the device
  (sampler alone and whole graph), and by the host sampler;
* BarabasiAlbert(1e7, m0=4, m=4), with its number of rounds;
* one order-30 Heat filter of 32 float32 signals on that BA graph.

Every time is a host clock around work that ends in a device synchronise, after one warm-up
run of the same shape.  The card's name, power limit and SM clock are printed with them.
"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def timed(fn, reps, sync):
    fn()
    sync()
    out = []
    for _ in range(reps):
        t = time.perf_counter()
        res = fn()
        sync()
        out.append(time.perf_counter() - t)
        del res
    return out


def show(name, ts, extra=""):
    print("%-34s median %9.2f ms  (%s)%s" % (name, 1e3 * float(np.median(ts)),
                                              ", ".join("%.2f" % (1e3 * t) for t in ts), extra))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--skip-host", action="store_true")
    args = ap.parse_args()
    import torch
    import pygsp_b200 as gsp
    from pygsp_b200.graphs import random_graphs as rg
    from pygsp_b200.graphs.generators import _sbm_blocks, sbm_adjacency

    try:
        print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm",
                              "--format=csv"], capture_output=True, text=True).stdout.strip())
    except OSError:
        print("nvidia-smi not available")
    sync = torch.cuda.synchronize

    N, k, p, q, seed = 10 ** 7, 8, 5e-6, 5e-7, 0
    rng = np.random.default_rng(seed)
    z, M = _sbm_blocks(rng, N, k, None, p, q)
    key = int(rng.integers(2 ** 63))
    W = rg.sbm_device(N, k, z, M, False, False, key)
    print("SBM config 4: nnz(W) = %d" % W.nnz)
    del W
    show("SBM device, sampler + from_coo", timed(
        lambda: rg.sbm_device(N, k, z, M, False, False, key), args.reps, sync))
    show("SBM device, whole StochasticBlockModel", timed(
        lambda: gsp.graphs.StochasticBlockModel(N, k=k, p=p, q=q, seed=seed, backend="device"),
        args.reps, sync))
    if not args.skip_host:
        t = time.perf_counter()
        Wh, _ = sbm_adjacency(N, k, None, p, q, seed=seed)
        show("SBM host sampler (sbm_adjacency)", [time.perf_counter() - t],
             "  nnz %d" % Wh.nnz)
        del Wh

    bkey = int(np.random.default_rng(seed).integers(2 ** 63))
    _, rounds = rg.barabasi_albert_device(10 ** 7, 4, 4, bkey)
    show("BarabasiAlbert(1e7, 4, 4)", timed(
        lambda: rg.barabasi_albert_device(10 ** 7, 4, 4, bkey), args.reps, sync),
        "  rounds %d" % rounds)

    B = gsp.graphs.BarabasiAlbert(10 ** 7, m0=4, m=4, seed=seed)
    deg = torch.diff(B.W.indptr)
    print("BA graph: nnz(W) = %d, max degree %d" % (B.W.nnz, int(deg.max())))
    B.estimate_lmax()
    g = gsp.filters.Heat(B, scale=50)
    x = torch.from_numpy(np.random.default_rng(0).standard_normal((B.N, 32)).astype(np.float32)
                         ).cuda()
    show("Heat order 30, 32 signals, BA 1e7", timed(lambda: g.filter(x, order=30), args.reps,
                                                    sync))


if __name__ == "__main__":
    main()
