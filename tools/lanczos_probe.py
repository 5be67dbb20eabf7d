"""Timings of Lanczos filtering (filters.lanczos_op, csrc/krylov.cu) on BASELINE config 2.

    python tools/lanczos_probe.py [--orders 10 30 60] [--nsig 64] [--reps 5] [--out DIR]

Graph: Sensor(1e6, k=10, seed=0, order='morton'), float32, Heat(scale=50).  For each order it
reports the end-to-end call time (CUDA events around the call, median and every one of --reps
after one warm-up; all orders are timed before the profiler is first started), the host time of
the per-column eigendecompositions, and, from a separate torch.profiler run, the device time split
into the SpMM, the reorthogonalisation (per-column Gram and update), the other Lanczos kernels,
the combine and any other kernel (listed by name).
The byte model is (m^2 + 7m) passes over one (N, nsig) signal block for order m (full
reorthogonalisation reads the basis twice per step); its time at the data-sheet 3.35 TB/s over
the measured Lanczos time is reported as the achieved fraction of that model.
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


def category(name):
    if "cheby_step" in name:
        return "spmm"
    if "krylov_cgs" in name:
        return "reorth"
    if "krylov_combine" in name:
        return "combine"
    if "krylov" in name or "sum_parts" in name:          # sum_parts: the Krylov partials sums
        return "other_lanczos"
    return "other"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--orders", type=int, nargs="+", default=[10, 30, 60])
    ap.add_argument("--nsig", type=int, default=64)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import numpy as np
    import torch
    import pygsp_b200 as gsp
    G = gsp.graphs.Sensor(1_000_000, k=10, seed=0, order="morton", dtype=np.float32)
    f = gsp.filters.Heat(G, scale=50)
    gen = torch.Generator(device=G.device).manual_seed(0)
    X = torch.randn((G.N, a.nsig), generator=gen, device=G.device, dtype=torch.float32)
    block = G.N * a.nsig * 4
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    rows = []
    coeff = gsp.filters.compute_cheby_coeff(f, m=30)
    gsp.filters.cheby_op(G, coeff, X)
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    cheb = []
    for _ in range(a.reps):
        t0.record()
        gsp.filters.cheby_op(G, coeff, X)
        t1.record()
        t1.synchronize()
        cheb.append(t0.elapsed_time(t1))
    # all timings first, with the profiler never started in this process before them
    import time
    from pygsp_b200.filters import approximations as approx
    host = []
    coefficients = approx._lanczos_coefficients

    def timed_coefficients(*args):
        t = time.perf_counter()
        W = coefficients(*args)
        host.append((time.perf_counter() - t) * 1e3)
        return W
    approx._lanczos_coefficients = timed_coefficients
    calls = {}
    for m in a.orders:
        gsp.filters.lanczos_op(f, X, order=m)                 # warm-up
        torch.cuda.synchronize()
        times = []
        del host[:]
        for _ in range(a.reps):
            t0.record()
            gsp.filters.lanczos_op(f, X, order=m)
            t1.record()
            t1.synchronize()
            times.append(t0.elapsed_time(t1))
        calls[m] = (times, statistics.median(host[-a.reps:]))
    approx._lanczos_coefficients = coefficients
    from torch.profiler import ProfilerActivity, profile
    for m in a.orders:
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            gsp.filters.lanczos_op(f, X, order=m)
            torch.cuda.synchronize()
        split, other = {}, {}
        for ev in prof.key_averages():
            t = getattr(ev, "device_time_total", None)
            if t is None:
                t = ev.cuda_time_total
            if t:
                c = category(ev.key)
                split[c] = split.get(c, 0.0) + t / 1e3
                if c == "other":
                    other[ev.key[:60]] = round(t / 1e3, 3)
        times, host_ms = calls[m]
        ms = statistics.median(times)
        model = (m * m + 7 * m) * block
        rows.append({"order": m, "call_ms": round(ms, 2),
                     "call_ms_all": [round(t, 2) for t in times],
                     "host_coefficients_ms": round(host_ms, 2),
                     "device_ms": {k: round(v, 2) for k, v in split.items()},
                     "device_ms_total": round(sum(split.values()), 2), "other_kernels": other,
                     "model_GB": round(model / 1e9, 1),
                     "model_ms_at_peak": round(model / PEAK * 1e3, 1),
                     "fraction_of_model": round(model / PEAK * 1e3 / ms, 3)})
        print(json.dumps(rows[-1]), flush=True)
    clocks = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,clocks.max.sm,power.draw",
                             "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    res = {"gpu": gpu, "clocks_after": clocks, "N": G.N, "nsig": a.nsig, "cheby30_ms": round(statistics.median(cheb), 2),
           "rows": rows}
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "lanczos_probe.json"), "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
