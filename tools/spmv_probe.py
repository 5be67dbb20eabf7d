"""SpMV (Lanczos operator) timing on the bench graph, L2-warm and L2-cold (needs a GPU).

    python tools/spmv_probe.py [--n 1000000]

Variants are selected through GSPB200_SPMV / GSPB200_SPMV_TR (read per launch).  Warm: 50
back-to-back products (x, indptr and most of the CSR stay in the 50 MB L2, as inside
Lanczos); cold: a 512 MB memset between products.  One JSON line per variant.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    a = ap.parse_args()
    import torch
    import bench
    import pygsp_b200 as gsp
    G = gsp.graphs.Sensor(a.n, k=10, seed=0, order="morton")
    L = G.L
    x = torch.randn(G.N, 1, device="cuda")
    flush = torch.empty(512 << 20, dtype=torch.uint8, device="cuda")
    peak, _ = bench.measured_peak()
    nbytes = 8 * L.nnz + 4 * (G.N + 1) + 8 * G.N
    ref = None
    for name, env in (("subwarp", {}), ("subwarp_lpr16", {"SPMV_LPR": "16"}), ("subwarp_lpr4", {"SPMV_LPR": "4"}),
                      ("window", {"SPMV": "window"}), ("window_tr128", {"SPMV": "window", "SPMV_TR": "128"})):
        for k, v in env.items():
            os.environ["GSPB200_" + k] = v
        y = L.dot(x)
        torch.cuda.synchronize()
        if ref is None:
            ref = y.clone()
        err = float((y - ref).abs().max() / ref.abs().max())
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(50):
            L.dot(x)
        e.record()
        torch.cuda.synchronize()
        warm = s.elapsed_time(e) / 50 * 1e3
        cold = []
        for _ in range(10):
            flush.zero_()
            s.record()
            L.dot(x)
            e.record()
            torch.cuda.synchronize()
            cold.append(s.elapsed_time(e) * 1e3)
        cold_us = sorted(cold)[len(cold) // 2]
        print(json.dumps({"variant": name, "warm_us": round(warm, 2), "cold_us": round(cold_us, 2),
                          "cold_frac_of_hbm": round(nbytes / cold_us / 1e3 / peak, 3),
                          "warm_GBps": round(nbytes / warm / 1e3, 1), "rel_diff_vs_first": err,
                          "algorithmic_bytes": nbytes}), flush=True)
        for k in env:
            del os.environ["GSPB200_" + k]


if __name__ == "__main__":
    main()
