"""Time per iteration of learning.classification_tikhonov_simplex (csrc/simplex.cu).

    python tools/simplex_probe.py [--classes 2 4 10 32] [--reps 3] [--out DIR]

Graph: Sensor(1e6, k=10, seed=0, order='morton'), float32 and float64; 5 % of the vertices
labelled with seeded random classes, tau = 1.  The time per iteration is the difference of two
fixed-length runs (rtol=None, maxit=20 and maxit=220), each timed by CUDA events around the call
after one warm-up run of the same shape, divided by 200: set-up and the per-batch reads of the
stop record cancel.  Median of --reps.

Byte model per iteration, from the shapes: the CSR of L once (nnz (4 + s) + 4 (N + 1)), the
SpMM's read of X_k and write of L X_k (2 N C s, the gather's reuse assumed to hit in cache), and
the row pass's reads of X_k, X_{k-1}, L X_k, L X_{k-1} and the labels and its write of x_{k+1}
(5 N C s + 4 N), s = 4 or 8 bytes.  Its time at the data-sheet 3.35 TB/s over the measured time
is the achieved fraction.  The card's name and power limit are read in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
PEAK = 3.35e12
K1, K2 = 20, 220


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--classes", type=int, nargs="+", default=[2, 4, 10, 32])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import numpy as np
    import torch
    import pygsp_b200 as gsp
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    rows = []
    for dtype in (np.float32, np.float64):
        G = gsp.graphs.Sensor(1_000_000, k=10, seed=0, order="morton", dtype=dtype)
        G.estimate_lmax()
        s = np.dtype(dtype).itemsize
        n, nnz = G.N, G.L.nnz
        rng = np.random.default_rng(0)
        M = rng.uniform(size=n) < 0.05
        for C in a.classes:
            y = rng.integers(0, C, n).astype(np.float64)
            y[0], M[0] = C - 1, True
            y_dev = torch.as_tensor(y, device=G.device)

            def timed(k):
                t0 = torch.cuda.Event(enable_timing=True)
                t1 = torch.cuda.Event(enable_timing=True)
                t0.record()
                gsp.learning.classification_tikhonov_simplex(G, y_dev, M, tau=1.0, rtol=None,
                                                             maxit=k, verbosity="NONE")
                t1.record()
                torch.cuda.synchronize()
                return t0.elapsed_time(t1) * 1e-3

            timed(K1)
            timed(K2)
            per_it = statistics.median((timed(K2) - timed(K1)) / (K2 - K1) for _ in range(a.reps))
            model = nnz * (4 + s) + 4 * (n + 1) + 7 * n * C * s + 4 * n
            rows.append({"dtype": np.dtype(dtype).name, "classes": C, "n": n, "nnz": nnz,
                         "us_per_iteration": per_it * 1e6, "model_bytes": model,
                         "fraction_of_3.35TBps": model / PEAK / per_it, "gpu": gpu})
            print(json.dumps(rows[-1]), flush=True)
        del G
        torch.cuda.empty_cache()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "simplex_probe.json"), "w") as fh:
            json.dump(rows, fh, indent=1)


if __name__ == "__main__":
    main()
