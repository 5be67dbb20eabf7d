"""Timings of the graph features (pygsp_b200/features.py, csrc/moments.cu).

    python tools/features_probe.py [--n 100000] [--M 100] [--order 30] [--reps 3]
                                   [--widths 32 64 128] [--naive-chunks 4] [--out DIR]

Graph: Sensor(n, k=10, seed=0, order='morton'), float32, lmax estimated once.  Reports, with
CUDA events around each call (median of --reps after one warm-up):
  * compute_spectrogram(G, M) end to end;
  * cheby_moments_device at each probe width, with the byte model
    ceil(N/b) m (8 nnz + 4 (N + 1) + 5 N b 4) -- per step the CSR, the step's gather of x_cur and
    its read of x_old and write of x_new, and the moment pass's two reads -- and that model's time
    at the data-sheet 3.35 TB/s over the measured time;
  * the naive route for comparison: for each probe block, M separate single-filter Clenshaw
    filterings of the identity columns plus their column norms, timed on --naive-chunks blocks of
    128 columns and extrapolated to ceil(N/128) blocks;
  * compute_avg_adj_deg.
"""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
PEAK = 3.35e12


def timed(fn, reps):
    import torch
    fn()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    out = []
    for _ in range(reps):
        t0.record()
        fn()
        t1.record()
        t1.synchronize()
        out.append(t0.elapsed_time(t1))
    return statistics.median(out), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=100_000)
    ap.add_argument("--M", type=int, default=100)
    ap.add_argument("--order", type=int, default=30)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--widths", type=int, nargs="+", default=[32, 64, 128])
    ap.add_argument("--naive-chunks", type=int, default=4)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import numpy as np
    import torch
    import pygsp_b200 as gsp
    from pygsp_b200 import _native as nat
    from pygsp_b200.filters import approximations as approx
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                          "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    G = gsp.graphs.Sensor(a.n, k=10, seed=0, order="morton", dtype=np.float32)
    G.estimate_lmax()
    L, lmax, n, m = G.L, G.lmax, G.N, a.order
    res = {"gpu": gpu, "N": n, "nnz": L.nnz, "M": a.M, "order": m}
    ms, all_ms = timed(lambda: gsp.features.compute_spectrogram(G, M=a.M, order=m), a.reps)
    res["spectrogram_ms"], res["spectrogram_ms_all"] = round(ms, 1), [round(t, 1) for t in all_ms]
    print(json.dumps(res), flush=True)
    rows = []
    for b in a.widths:
        ms, all_ms = timed(lambda: approx.cheby_moments_device(L, lmax, m, width=b), a.reps)
        model = math.ceil(n / b) * m * (8 * L.nnz + 4 * (n + 1) + 5 * n * b * 4)
        rows.append({"width": b, "moments_ms": round(ms, 1),
                     "moments_ms_all": [round(t, 1) for t in all_ms],
                     "model_GB": round(model / 1e9, 1),
                     "model_ms_at_peak": round(model / PEAK * 1e3, 1),
                     "fraction_of_peak": round(model / PEAK * 1e3 / ms, 3)})
        print(json.dumps(rows[-1]), flush=True)
    res["moments"] = rows
    # naive route: M Clenshaw filterings per block of 128 identity columns
    b = 128
    scale = np.linspace(0, lmax, a.M)
    coeffs = [approx.compute_cheby_coeff(
        gsp.filters.Filter(G, lambda x, s=s: np.exp(-a.M * ((x - s) / lmax) ** 2)), m=m)
        for s in scale]
    X = torch.empty((n, b), dtype=torch.float32, device=G.device)
    out = torch.empty((n, b), dtype=torch.float32, device=G.device)
    work = torch.empty((2, n, b), dtype=torch.float32, device=G.device)
    sq = torch.empty((a.M, b), dtype=torch.float64, device=G.device)

    def naive():
        for q in range(a.naive_chunks):
            with torch.cuda.device(G.device):
                nat.call("gsp_probe_block_f32", nat.i64(n), nat.i64(q * b), nat.i64(b), X,
                         nat.stream_ptr(G.device))
            for j, c in enumerate(coeffs):
                approx.cheby_clenshaw_device(L, lmax, c, X, out=out, work=work)
                sq[j] = (out.double() ** 2).sum(dim=0)
    ms, all_ms = timed(naive, 1)
    blocks = math.ceil(n / b)
    res["naive_ms_per_block"] = round(ms / a.naive_chunks, 1)
    res["naive_ms_extrapolated"] = round(ms / a.naive_chunks * blocks, 0)
    print(json.dumps({"naive_ms_per_block": res["naive_ms_per_block"],
                      "naive_ms_extrapolated": res["naive_ms_extrapolated"]}), flush=True)
    ms, all_ms = timed(lambda: gsp.features.compute_avg_adj_deg(G), a.reps)
    res["avg_adj_deg_ms"] = round(ms, 2)
    res["clocks_after"] = subprocess.run(
        ["nvidia-smi", "--query-gpu=clocks.sm,clocks.max.sm,power.draw", "--format=csv,noheader"],
        capture_output=True, text=True).stdout.strip()
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "features_probe.json"), "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
