"""Timing of the differential operator on BASELINE config 2 (needs a GPU).

    python tools/difference_probe.py [--n 1000000] [--reps 20] [--out FILE]

One JSON line per measurement (also appended to --out when given):
  card   : GPU name, power limit and SM clock limit (nvidia-smi), read in the same run;
  build  : compute_differential_operator() on the config-2 graph (Sensor-type k-NN, 1e6
           vertices, k = 10, Morton order, float32), milliseconds after a warm-up build;
  grad / div at 1 and 64 signals: milliseconds per product from CUDA events (after warm-up)
           and the achieved bytes/s against the byte model below, computed from the shapes:
             grad: 4 (Ne + 1) + 8 nnz(D^T) + 4 N Nsig + 4 Ne Nsig
             div : 4 (N + 1)  + 8 nnz(D)   + 4 Ne Nsig + 4 N Nsig
           (indptr, indices + values, input block read once, output block written once).
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_PEAK = 3.35e12          # H100 SXM data sheet


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
    import torch
    for _ in range(3):
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
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("difference_probe needs a CUDA device")
    import pygsp_b200 as gsp
    emit(dict(kind="card", card=card(), torch=torch.__version__), a.out)

    G = gsp.graphs.Sensor(a.n, k=10, seed=0, order="morton")
    ms = timed(G.compute_differential_operator, max(3, a.reps // 4))
    D = G.D
    n, ne = G.N, G.Ne
    emit(dict(kind="build", graph="config2", n=n, n_edges=ne, nnz_D=D.nnz, ms=round(ms, 3)),
         a.out)
    gen = torch.Generator(device=G.device).manual_seed(0)
    for nsig in (1, 64):
        shape_x = (n,) if nsig == 1 else (n, nsig)
        shape_y = (ne,) if nsig == 1 else (ne, nsig)
        x = torch.randn(shape_x, generator=gen, device=G.device, dtype=G.dtype)
        y = torch.randn(shape_y, generator=gen, device=G.device, dtype=G.dtype)
        cases = {
            "grad": (lambda: G.grad(x), 4 * (ne + 1) + 8 * D.T.nnz + 4 * n * nsig + 4 * ne * nsig),
            "div": (lambda: G.div(y), 4 * (n + 1) + 8 * D.nnz + 4 * ne * nsig + 4 * n * nsig),
        }
        for name, (fn, nbytes) in cases.items():
            t = timed(fn, a.reps)
            emit(dict(kind=name, nsig=nsig, ms=round(t, 4), model_bytes=nbytes,
                      gbps=round(nbytes / (t / 1e3) / 1e9, 1),
                      share_of_peak=round(nbytes / (t / 1e3) / HBM_PEAK, 3)), a.out)


if __name__ == "__main__":
    main()
