"""Timing of kron_reduction(method='walks') and of graph_multiresolution with walks and sketched
resistances (needs a GPU).

    python tools/kron_walks_probe.py [--reps 3] [--sizes 10000,30000,100000] [--out FILE]

One JSON line per measurement (also appended to --out when given):
  card     : GPU name, power limit and SM clock limit (nvidia-smi), read in the same run;
  kron     : kron_reduction of Sensor(10^4)'s eigenvector split, 'exact' against 'walks' (16
             samples): total ms, entries of the result, and for the walks
             walk_ms     -- gsp_schur_walk_f64 (every item),
             assembly_ms -- DeviceCSR.from_coo of the exact and sampled triplets,
             steps mean / p99 / max per item (both walks of an item);
  pipeline : graph_multiresolution(Sensor(N, k=10, seed=1, order='morton'), 3,
             kron_method='walks', resistances='sketch') at every size: total ms, split into
             kron_ms (the levels' reductions), kreg_ms (K_reg), sparsify_ms (graph_sparsify) and
             other_ms (eigenvectors, estimate_lmax, filters), with the levels' N and entries.
Times are milliseconds, host clock around work that ends in a device synchronise; the median of
--reps calls after one warm-up call (sizes above 3 10^4 are called once after the warm-up of the
smaller ones).
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

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


def timed(torch, fn, *args, **kw):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn(*args, **kw)
    torch.cuda.synchronize()
    return out, 1e3 * (time.perf_counter() - t0)


class Wrap:
    """Adds the time of every call of ``module.name`` to ``acc[key]`` while installed."""

    def __init__(self, torch, module, name, acc, key):
        self.torch, self.module, self.name, self.acc, self.key = torch, module, name, acc, key
        self.fn, self.raw = getattr(module, name), vars(module)[name]

    def __enter__(self):
        def wrapped(*args, **kw):
            out, ms = timed(self.torch, self.fn, *args, **kw)
            self.acc[self.key] = self.acc.get(self.key, 0.0) + ms
            return out
        setattr(self.module, self.name, wrapped)
        return self

    def __exit__(self, *exc):
        setattr(self.module, self.name, self.raw)


def kron_split(gsp, torch, G, ind):
    red = gsp.reduction
    from pygsp_b200.graphs import csr
    acc, stats = {}, {}
    call0 = red._call

    def call(name, *args):
        if name != "gsp_schur_walk_f64":
            return call0(name, *args)
        _, ms = timed(torch, call0, name, *args)
        acc["walk_ms"] = acc.get("walk_ms", 0.0) + ms

    red._call = call
    try:
        M = red._device_matrix(G.L, G.device)
        ex = torch.zeros(G.N, dtype=torch.float64, device=G.device)
        with Wrap(torch, csr.DeviceCSR, "from_coo", acc, "assembly_ms"):
            H, total = timed(torch, red._schur_walks, M, ind, 16, red._sampling_seed(0, 1 << 21),
                             2 ** 20, excess=ex, stats=stats)
    finally:
        red._call = call0
    # induced() assembles through from_counts: the one from_coo is the final sum of the triplets
    s = stats["steps"].double()
    return H, total, acc, {"mean": float(s.mean()), "p99": float(torch.quantile(s[:2 ** 24], 0.99)),
                           "max": int(s.max())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--sizes", default="10000,30000,100000")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    import pygsp_b200 as gsp
    red = gsp.reduction
    emit({"card": card()}, a.out)

    G = gsp.graphs.Sensor(10_000, k=10, seed=1, order="morton")
    V = G._largest_eigenvector(seed=0)
    V *= np.sign(V[0])
    ind = np.nonzero(V >= 0)[0]
    rec = {"kron": "Sensor(1e4) eigenvector split", "kept": int(ind.size)}
    ex_ms, wk = [], []
    for r in range(a.reps + 1):
        E, ms = timed(torch, red.kron_reduction, G, ind)
        if r:
            ex_ms.append(ms)
        H, total, acc, steps = kron_split(gsp, torch, G, ind)
        if r:
            wk.append((total, acc))
    rec["exact_ms"] = statistics.median(ex_ms)
    rec["exact_entries"] = int(E.W.nnz)
    rec["walks_ms"] = statistics.median(t for t, _ in wk)
    rec["walk_ms"] = statistics.median(acc["walk_ms"] for _, acc in wk)
    rec["assembly_ms"] = statistics.median(acc["assembly_ms"] for _, acc in wk)
    rec["walks_offdiag_entries"] = int(H.nnz - H.shape[0])
    rec["steps"] = steps
    emit(rec, a.out)

    for n in [int(x) for x in a.sizes.split(",")]:
        reps = a.reps if n <= 30_000 else 1
        runs = []
        for r in range(reps + (1 if n <= 30_000 else 0)):
            G = gsp.graphs.Sensor(n, k=10, seed=1, order="morton")
            acc = {}
            with Wrap(torch, red, "_kron_graph", acc, "kron_ms"), \
                    Wrap(torch, red, "_kron_regularized", acc, "kreg_ms"), \
                    Wrap(torch, red, "graph_sparsify", acc, "sparsify_ms"):
                Gs, total = timed(torch, red.graph_multiresolution, G, 3, kron_method="walks",
                                  resistances="sketch")
            if r or n > 30_000:
                acc["total_ms"] = total
                runs.append(acc)
        rec = {"pipeline": "Sensor(%d)" % n, "N": [g.N for g in Gs],
               "entries": [int(g.W.nnz) for g in Gs], "reps": len(runs)}
        for k in ("total_ms", "kron_ms", "kreg_ms", "sparsify_ms"):
            rec[k] = statistics.median(x[k] for x in runs)
        rec["other_ms"] = rec["total_ms"] - rec["kron_ms"] - rec["kreg_ms"] - rec["sparsify_ms"]
        rec["connected"] = all(g.is_connected() for g in Gs)
        emit(rec, a.out)


if __name__ == "__main__":
    main()
