"""Time per iteration of optimization.prox_tv (csrc/tv.cu).

    python tools/tv_probe.py [--nsig 1 8 64] [--reps 3] [--out DIR]

Graph: Sensor(1e6, k=10, seed=0, order='morton') (config 2), float32 and float64, the fused
path (A = None) and the A = identity path (Python-driven: D u, At, the axpy, A, edge pass),
alternated within each repetition.  The time per iteration is the difference of two fixed-length
runs (tol=0, maxit=20 and maxit=220), each timed by CUDA events around the call after one
warm-up run of the same shape, divided by 200: set-up, the final vertex pass and the per-batch
reads of the stop record cancel.  Median of --reps.

Byte model per iteration of the fused path, from the shapes (s = 4 or 8 bytes per value):
  vertex pass  the CSR of D (4 (N + 1) + nnz_D (4 + s)), the gather of u (Ne Nsig s, each row
               once), u's own row, x_old = x and the write of z (3 N Nsig s);
  edge pass    the CSR of D^T (4 (Ne + 1) + nnz_D (4 + s)), the gather of z (N Nsig s, each row
               once), u_k, u_{k-1}, g_{k-1} in and g_k, u_{k+1} out (5 Ne Nsig s), and the vertex
               slice's x and z (2 N Nsig s).
Its time at the data-sheet 3.35 TB/s over the measured time is the achieved fraction.  The card's
name and power limit are read in the same run.  With --oracle the CPU oracle's time per iteration
at 1e5 vertices is printed too (a CPU number).
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
PEAK = 3.35e12
K1, K2 = 20, 220


def model_bytes(n, ne, nnz_d, nsig, s):
    vertex = 4 * (n + 1) + nnz_d * (4 + s) + ne * nsig * s + 3 * n * nsig * s
    edge = 4 * (ne + 1) + nnz_d * (4 + s) + n * nsig * s + 5 * ne * nsig * s + 2 * n * nsig * s
    return vertex + edge


def ptxas_counts():
    """Registers, spills and shared memory of the new kernels, from -Xptxas -v."""
    from pygsp_b200 import build
    out = subprocess.run([build._nvcc(), "-O3", "-std=c++17", *build.ARCH, "-Xptxas", "-v",
                          "-I", os.path.join(ROOT, "include"), "-I", build.CSRC, "-c",
                          os.path.join(build.CSRC, "tv.cu"), "-o", os.devnull],
                         capture_output=True, text=True)
    lines, name, rows = out.stderr.splitlines(), None, []
    for ln in lines:
        if "Compiling entry function" in ln:
            name = ln.split("'")[1]
        elif name and "Used" in ln and "registers" in ln and "tv_edge_kernel" in name:
            rows.append((name, ln.split("info    :")[-1].strip()))
        elif name and "spill" in ln and "tv_edge_kernel" in name:
            rows.append((name, ln.strip()))
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nsig", type=int, nargs="+", default=[1, 8, 64])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--n", type=int, default=10 ** 6)
    ap.add_argument("--oracle", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import numpy as np
    import torch
    import pygsp_b200 as gsp
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print("card:", gpu)
    for name, line in ptxas_counts():
        print("ptxas %s: %s" % (name, line))
    results = []
    graphs = {}
    for dt in (np.float32, np.float64):
        G = gsp.graphs.Sensor(a.n, k=10, seed=0, order="morton", dtype=dt)
        G.estimate_lmax()
        G.compute_differential_operator()
        graphs[dt] = G
    ident = (lambda v: v)

    def run(G, x, maxit, A):
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        start.record()
        gsp.optimization.prox_tv(x, 0.1, G, A=A, At=A, tol=0, maxit=maxit)
        end.record()
        torch.cuda.synchronize()
        return start.elapsed_time(end) * 1e-3

    for nsig in a.nsig:
        for dt, G in graphs.items():
            x = torch.randn(G.N, nsig, dtype=G.dtype, device="cuda",
                            generator=torch.Generator("cuda").manual_seed(0))
            for A in (None, ident):
                run(G, x, K1, A)
                run(G, x, K2, A)
            per = {None: [], "identity": []}
            for _ in range(a.reps):
                for A, key in ((None, None), (ident, "identity")):
                    per[key].append((run(G, x, K2, A) - run(G, x, K1, A)) / (K2 - K1))
            s = np.dtype(dt).itemsize
            byt = model_bytes(G.N, G.Ne, G.D.nnz, nsig, s)
            for key, ts in per.items():
                t = statistics.median(ts)
                row = {"path": "fused" if key is None else "A=identity", "dtype": np.dtype(dt).name,
                       "nsig": nsig, "N": G.N, "Ne": G.Ne, "ms_per_iter": t * 1e3,
                       "model_bytes": byt, "fraction_of_3.35TB/s": byt / PEAK / t,
                       "spread_ms": [round(v * 1e3, 4) for v in ts]}
                results.append(row)
                print(json.dumps(row))
    if a.oracle:
        from scipy import sparse
        from oracle import optimization_oracle as oo
        G = gsp.graphs.Sensor(10 ** 5, k=10, seed=0, order="morton", dtype=np.float64)
        D = G.D.to_scipy_csc()
        x = np.random.default_rng(0).normal(size=(G.N, 1))
        t0 = time.perf_counter()
        oo.prox_tv_fgp(x, 0.1, sparse.csc_matrix(D), G.lmax, tol=0, maxit=20)
        t = (time.perf_counter() - t0) / 21
        row = {"path": "CPU oracle (NumPy/SciPy, float64)", "N": G.N, "nsig": 1,
               "ms_per_iter": t * 1e3}
        results.append(row)
        print(json.dumps(row))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "tv_probe.json"), "w") as fh:
            json.dump({"card": gpu, "rows": results}, fh, indent=1)


if __name__ == "__main__":
    main()
