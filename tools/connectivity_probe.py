"""Timing of the connectivity methods (needs a GPU).

    python tools/connectivity_probe.py [--n 1000000] [--reps 5] [--out FILE]

One JSON line per measurement (also appended to --out when given):
  card  : GPU name, power limit and SM clock limit (nvidia-smi), read in the same run;
  graph : the two inputs, float32 --
            config2 : BASELINE config 2, Sensor-type k-NN graph, 1e6 vertices, k = 10, Morton order;
            sbm     : StochasticBlockModel(1e6, k=8, p=5e-5, q=5e-6, seed=0), config 4's mean degree;
  call  : milliseconds per call (median of --reps after one warm-up call, host clock around
          calls that end in a device synchronise) of
            is_connected           undirected (union-find; the cache is cleared before each call)
            is_connected_directed  on a directed variant: W's structure with the weights above
                                   the diagonal doubled (frontier BFS through W and W^T)
            extract_components
            subgraph_sorted / subgraph_shuffled   a seeded random half of the vertices, sorted
                                   or in random order (a CUDA tensor of ids)
"""
import argparse
import json
import os
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


def timed(fn, reps):
    import numpy as np
    import torch
    fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        times.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(times))


def directed_variant(gsp, G):
    """W's structure with the weights above the diagonal doubled, built on the device."""
    import torch
    W = G.W
    rows = gsp.graphs.csr.row_ids(W.indptr)
    data = torch.where(W.indices > rows, W.data * 2, W.data)
    return gsp.graphs.Graph(gsp.graphs.DeviceCSR(W.indptr, W.indices, data, W.shape))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("connectivity_probe needs a CUDA device")
    import pygsp_b200 as gsp
    emit(dict(kind="card", card=card(), torch=torch.__version__), a.out)

    inputs = {
        "config2": lambda: gsp.graphs.Sensor(a.n, k=10, seed=0, order="morton"),
        "sbm": lambda: gsp.graphs.StochasticBlockModel(a.n, k=8, p=5e-5, q=5e-6, seed=0),
    }
    for name, make in inputs.items():
        G = make()
        Gd = directed_variant(gsp, G)
        labels, n_comp = G._component_labels(False)
        emit(dict(kind="graph", graph=name, n=G.N, nnz=G.W.nnz,
                  components=int(n_comp.item()), directed_variant=Gd.is_directed()), a.out)
        half = np.random.default_rng(0).permutation(G.N)[:G.N // 2]
        half_sorted = np.sort(half)
        half_dev = torch.as_tensor(half, device=G.device)

        def connected():
            G._connected = None
            return G.is_connected()

        def connected_directed():
            Gd._connected = None
            return Gd.is_connected()
        calls = {
            "is_connected": connected,
            "is_connected_directed": connected_directed,
            "extract_components": G.extract_components,
            "subgraph_sorted": lambda: G.subgraph(half_sorted),
            "subgraph_shuffled": lambda: G.subgraph(half_dev),
        }
        for call, fn in calls.items():
            emit(dict(kind="call", graph=name, call=call, ms=round(timed(fn, a.reps), 3)), a.out)
        emit(dict(kind="result", graph=name, connected=connected(),
                  connected_directed=connected_directed()), a.out)
        del G, Gd


if __name__ == "__main__":
    main()
