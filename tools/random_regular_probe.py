"""Timing of RandomRegular (needs a GPU).

    python tools/random_regular_probe.py [--reps 3] [--out FILE]

One JSON line per measurement (also appended to --out when given):
  card           : GPU name, power limit and SM clock limit (nvidia-smi), read in the same run;
  random_regular : RandomRegular(N, k=10) for N = 10**6 and 10**7, float32: the whole constructor
                   (sampler, assembly, Graph checks and Laplacian), the sampler call alone
                   (gsp_random_regular: rounds and tail) and DeviceCSR.from_coo of its output
                   alone; the attempts and rounds taken.  The split between the rounds and the
                   tail inside the sampler call is not measured.
Times are milliseconds, the median of --reps calls after one warm-up call, each call timed by
CUDA events around synchronised work.
"""
import argparse
import ctypes
import json
import os
import statistics
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


def median_ms(fn, reps):
    import torch
    fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        times.append(s.elapsed_time(e))
    return round(statistics.median(times), 3), [round(t, 3) for t in times]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import numpy as np
    import torch
    import pygsp_b200 as gsp
    from pygsp_b200 import _native as nat
    from pygsp_b200.graphs.csr import DeviceCSR

    torch.cuda.set_device(0)
    emit(dict(kind="card", card=card()), a.out)
    k, key = 10, 12345
    for N in (10 ** 6, 10 ** 7):
        rows = torch.empty(N * k, dtype=torch.int32, device="cuda")
        cols = torch.empty(N * k, dtype=torch.int32, device="cuda")
        att, rnd, ent = ctypes.c_int(0), ctypes.c_int(0), ctypes.c_int64(0)

        def sample():
            nat.call("gsp_random_regular", nat.i64(N), nat.i64(k), nat.i32(10), nat.u64(key),
                     rows, cols, nat.i32(0), ctypes.byref(att), ctypes.byref(rnd),
                     ctypes.byref(ent), nat.stream_ptr())
        ms_sample, all_sample = median_ms(sample, a.reps)
        ones = torch.ones(N * k, dtype=torch.float32, device="cuda")
        ms_coo, all_coo = median_ms(lambda: DeviceCSR.from_coo(rows, cols, ones, (N, N)), a.reps)
        del rows, cols, ones
        torch.cuda.empty_cache()
        ms_all, all_ctor = median_ms(lambda: gsp.graphs.RandomRegular(N=N, k=k, seed=0,
                                                                      dtype=np.float32), a.reps)
        G = gsp.graphs.RandomRegular(N=N, k=k, seed=0, dtype=np.float32)
        emit(dict(kind="random_regular", N=N, k=k, nnz=int(G.W.nnz), attempts=G._attempts,
                  rounds=G._rounds, sampler_attempts=att.value, sampler_rounds=rnd.value,
                  constructor_ms=ms_all, constructor_runs=all_ctor, sampler_ms=ms_sample,
                  sampler_runs=all_sample, from_coo_ms=ms_coo, from_coo_runs=all_coo,
                  rounds_vs_tail="not measured"), a.out)
        del G
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
