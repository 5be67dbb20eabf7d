"""Neighbour rings of the tiled Clenshaw steps: ring statistics (CPU) and per-launch kernel times
with the rings on and off (GPU).

    python tools/ring_probe.py cpu [--n 1000000 10000000] [--nsig 64]
    python tools/ring_probe.py gpu [--rounds 5] [--calls 10] [--variants VARIANT ...]

cpu: for the Morton k-NN graph of bench.py (host replica, k = 10) and each tile size R of
32 / 64 / 128: ring rows per tile (mean / p99 / max), runs per tile (mean / max), ring rows per
row owned, the stage bytes of the largest ring, and the CSR bytes a step streams without and with
rings (4-byte column id + 4-byte value, or 4-byte value + 2-byte ring position, per entry).

gpu: builds config 2 of bench.py once and runs, round-robin in one process, the Clenshaw call
under each variant -- GSPB200_* settings as NAME=VALUE[,NAME=VALUE], "base" for none; the library
reads them per call, and tile plans are kept per variant.  Per variant: ms per call from CUDA
events (profiler off), then one profiled call per round, from which the mean time of each launch
of cheby_step_tiled and cheby_pair_tiled is taken.  The card's name, power limit and SM clock are
read in the same process.  One JSON line per variant.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

DEFAULT_VARIANTS = ["TILE_RING=0,CLENSHAW_PAIRS=0", "TILE_RING=1,CLENSHAW_PAIRS=0",
                    "TILE_RING=0,CLENSHAW_PAIRS=1", "TILE_RING=1,CLENSHAW_PAIRS=1"]


def ring_stats(W, R):
    import ctypes
    from pygsp_b200 import _native as nat
    from oracle import pygsp_oracle as orc
    L = orc.laplacian(W.tocsr()).tocsr()
    L.sort_indices()
    n, T = L.shape[0], L.shape[0] // R
    indptr = np.ascontiguousarray(L.indptr, dtype=np.int32)
    indices = np.ascontiguousarray(L.indices, dtype=np.int32)
    count, ring_max = ctypes.c_int64(0), ctypes.c_int32(0)
    cap = L.nnz + T
    meta, runs = np.empty(4 * T, np.int32), np.empty(2 * cap, np.int32)
    local = np.empty(L.nnz, np.uint16)
    nat.call("gsp_cheby_ring_plan_host", nat.i64(n), indptr, indices, nat.i32(R), nat.i64(cap),
             meta, runs, local, ctypes.byref(count), ctypes.byref(ring_max))
    meta = meta.reshape(T, 4)
    size, nruns = meta[:, 2], meta[:, 1] - meta[:, 0]
    return {"R": R, "ring_rows_mean": round(float(size.mean()), 1),
            "ring_rows_p99": int(np.percentile(size, 99)), "ring_rows_max": int(ring_max.value),
            "runs_mean": round(float(nruns.mean()), 1), "runs_max": int(nruns.max()),
            "ring_per_row": round(float(size.mean()) / R, 3), "nnz": int(L.nnz)}


def cpu(a):
    import bench
    for n in a.n:
        W = bench.host_graph(n, 10, 0)
        for R in (32, 64, 128):
            st = ring_stats(W, R)
            st["N"] = n
            st["ring_stage_kb_max"] = round(st["ring_rows_max"] * 4 * a.nsig / 1024, 1)
            st["csr_mb_per_step"] = round(st["nnz"] * 8 / 1e6, 1)
            st["csr_mb_per_step_ring"] = round(st["nnz"] * 6 / 1e6, 1)
            print(json.dumps(st), flush=True)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip()


def gpu(a):
    import torch
    from torch.profiler import ProfilerActivity, profile
    import pygsp_b200 as gsp
    from pygsp_b200.filters import approximations as apx

    G = gsp.graphs.Sensor(a.n, k=10, seed=0, order="morton")
    G.estimate_lmax()
    g = gsp.filters.Heat(G, scale=50)
    c = np.atleast_2d(gsp.filters.compute_cheby_coeff(g, m=a.order))
    x = torch.randn(G.N, a.nsig, device="cuda", generator=torch.Generator("cuda").manual_seed(0))
    variants = a.variants or DEFAULT_VARIANTS
    plans = {v: {} for v in variants}
    ms = {v: [] for v in variants}
    kern = {v: {} for v in variants}
    clocks = []
    ref, same = None, {}

    def settings(v):
        return dict(kv.split("=") for kv in v.split(",") if kv and v != "base")

    for rnd in range(a.rounds + 1):                     # round 0: warm-up and plans
        for v in variants:
            env = settings(v)
            for k, val in env.items():
                os.environ["GSPB200_" + k] = val
            G.L._plans = plans[v]
            out = apx.cheby_clenshaw_device(G.L, G.lmax, c, x)
            torch.cuda.synchronize()
            if rnd == 0:
                ref = out.clone() if ref is None else ref
                same[v] = bool(torch.equal(out, ref))
            else:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(a.calls):
                    apx.cheby_clenshaw_device(G.L, G.lmax, c, x)
                e1.record()
                torch.cuda.synchronize()
                ms[v].append(e0.elapsed_time(e1) / a.calls)
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    apx.cheby_clenshaw_device(G.L, G.lmax, c, x)
                    torch.cuda.synchronize()
                for ev in prof.events():
                    for tag in ("cheby_step_tiled", "cheby_pair_tiled"):
                        if tag in ev.name and ev.device_type.name == "CUDA":
                            kern[v].setdefault(tag, []).append(ev.device_time / 1e3)
            for k in env:
                os.environ.pop("GSPB200_" + k, None)
        if rnd == 1:
            clocks.append(card())
    clocks.append(card())
    for v in variants:
        per = {t: {"launches_per_call": len(d) // a.rounds,
                   "ms_mean": round(float(np.mean(d)), 4), "ms_min": round(float(np.min(d)), 4),
                   "ms_max": round(float(np.max(d)), 4)} for t, d in kern[v].items()}
        print(json.dumps({"variant": v, "ms_per_call": [round(t, 3) for t in ms[v]],
                          "median_ms": round(float(np.median(ms[v])), 3), "kernels": per,
                          "same_bits_as_first_variant": same[v], "N": G.N, "nsig": a.nsig,
                          "order": a.order, "card": clocks}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("mode", choices=["cpu", "gpu"])
    ap.add_argument("--n", type=int, nargs="*", default=None)
    ap.add_argument("--nsig", type=int, default=64)
    ap.add_argument("--order", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--variants", nargs="*", default=None)
    a = ap.parse_args()
    if a.mode == "cpu":
        a.n = a.n or [1_000_000]
        cpu(a)
    else:
        a.n = (a.n or [1_000_000])[0]
        gpu(a)


if __name__ == "__main__":
    main()
