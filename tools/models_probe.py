"""Timing of the sampled graph models (needs a GPU).

    python tools/models_probe.py [--reps 3] [--out FILE]

One JSON line per measurement (also appended to --out when given):
  card       : GPU name, power limit and SM clock limit (nvidia-smi), read in the same run;
  community  : Community(N=10**6) with the default parameters (epsilon branch, about 500
               communities, world_density = 1/N), float32: the segmented radius count and fill
               alone, the inter-community subset draw alone, and the whole constructor (host
               coordinates, both searches, the draw, assembly and the Graph checks);
  swissroll  : SwissRoll(N=10**5) with the defaults, float32, the whole constructor.
Times are milliseconds per call from CUDA events after one warm-up call.
"""
import argparse
import json
import os
import subprocess
import sys

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


def timed(fn, reps, warmup=1):
    import torch
    for _ in range(warmup):
        fn()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(reps):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import numpy as np
    import torch
    import pygsp_b200 as gsp
    from pygsp_b200.graphs import sampled
    from pygsp_b200.graphs.random_graphs import RECT

    torch.cuda.set_device(0)
    emit(dict(kind="card", card=card()), a.out)

    N = 10 ** 6
    G = gsp.graphs.Community(N=N, seed=0, dtype=np.float32)
    sizes, eps = G.info["comm_sizes"], G.epsilon
    coords = torch.as_tensor(G.coords, device="cuda")
    start = np.concatenate([[0], np.cumsum(sizes)])
    inter = [(RECT, int(sizes[i] * sizes[j]), int(sizes[j]), int(start[i]), int(start[j]))
             for i in range(G.Nc) for j in range(i)]
    n_inter = int(G.world_density * (N ** 2 - np.sum(sizes ** 2)) / 2)
    ms_search = timed(lambda: sampled.radius_segments_device(coords, sizes, eps), a.reps)
    ms_draw = timed(lambda: sampled.subset_device(N, [(inter, n_inter)], 12345), a.reps)
    ms_all = timed(lambda: gsp.graphs.Community(N=N, seed=0, dtype=np.float32), a.reps)
    pairs = int(np.sum(sizes.astype(np.int64) ** 2))
    emit(dict(kind="community", N=N, Nc=int(G.Nc), nnz=int(G.W.nnz), n_inter=n_inter,
              segment_pairs=pairs, all_pairs=N * N, search_ms=round(ms_search, 3),
              inter_draw_ms=round(ms_draw, 3), constructor_ms=round(ms_all, 3)), a.out)

    M = 10 ** 5
    S = gsp.graphs.SwissRoll(N=M, seed=0, dtype=np.float32)
    ms_swiss = timed(lambda: gsp.graphs.SwissRoll(N=M, seed=0, dtype=np.float32), a.reps)
    emit(dict(kind="swissroll", N=M, nnz=int(S.W.nnz), constructor_ms=round(ms_swiss, 3)),
         a.out)


if __name__ == "__main__":
    main()
