"""Kernel-variant sweep on the bench workload (needs a GPU).

    python tools/sweep.py [--n 1000000] [--steps 5] VAR=VAL,VAR=VAL ...

Each positional argument is one configuration: a comma-separated list of
GSPB200_* environment overrides (without the prefix), e.g.
    KERNEL=rowgroup   TILE_R=32,TILE_S=3,TILE_NW=8,TILE_U=4
Prints ms per cheby_op call and the algorithmic HBM fraction for each.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--nsig", type=int, default=64)
    ap.add_argument("--nsigs", default=None, help="comma list: run every config for each width")
    ap.add_argument("--nscales", type=int, default=1)
    ap.add_argument("--order", type=int, default=30)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--graph", default="sensor", choices=["sensor", "grid2d"])
    ap.add_argument("--bank", default="heat", choices=["heat", "mexicanhat"])
    ap.add_argument("configs", nargs="*")
    a = ap.parse_args()
    import torch
    import bench
    import pygsp_b200 as gsp
    from pygsp_b200.filters import approximations as apx

    if a.graph == "grid2d":
        side = int(round(a.n ** 0.5))
        G = gsp.graphs.Grid2d(side, side)
        a.n = G.N
    else:
        G = gsp.graphs.Graph(bench.host_graph(a.n, 10, 0))
    G.estimate_lmax()
    if a.bank == "mexicanhat":
        filt = gsp.filters.MexicanHat(G, Nf=a.nscales)
    else:
        filt = gsp.filters.Heat(G, [50.0 / (i + 1) for i in range(a.nscales)])
    c = np.atleast_2d(np.array(gsp.filters.compute_cheby_coeff(filt, m=a.order)))
    print(json.dumps({"graph": a.graph, "N": G.N, "nnz_L": G.L.nnz, "lmax": G.lmax,
                      "lanczos_steps": G._lanczos_steps}), flush=True)
    peak, _ = bench.measured_peak()
    widths = [int(v) for v in a.nsigs.split(",")] if a.nsigs else [a.nsig]
    runs = [(w, cfg) for w in widths for cfg in (a.configs or ["KERNEL=rowgroup"])]
    ref, last_w = None, None
    for a.nsig, cfg in runs:
        if a.nsig != last_w:
            x = torch.randn(a.n, a.nsig, device="cuda",
                            generator=torch.Generator("cuda").manual_seed(0))
            _, _, b_call = bench.algorithmic_bytes(a.n, G.L.nnz, a.nsig, a.nscales, a.order)
            ref, last_w = None, a.nsig
        for k in [k for k in os.environ if k.startswith("GSPB200_")]:
            del os.environ[k]
        for kv in cfg.split(","):
            k, v = kv.split("=")
            os.environ["GSPB200_" + k] = v
        G.L._plans.clear()
        run = apx.cheby_op_device
        if os.environ.pop("GSPB200_CLENSHAW", None):
            run = lambda L_, lm, cc, xx: apx.cheby_clenshaw_device(L_, lm, cc[0], xx)[None]
        try:
            for _ in range(3):
                y = run(G.L, G.lmax, c, x)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.steps):
                y = run(G.L, G.lmax, c, x)
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / a.steps
            if ref is None:
                ref = y.clone()
            err = float((y - ref).abs().max() / ref.abs().max())
            plan = G.L.tile_plan(a.nsig, a.nscales)
            row = {"cfg": cfg, "nsig": a.nsig, "ms": round(ms, 3),
                   "frac": round(b_call / ms / 1e6 / peak, 4),
                   "units_per_s": a.n * a.nsig * a.order / ms * 1e3,
                   "maxdiff_vs_first": err, "plan": plan.as_dict() if plan else None}
        except Exception as exc:  # keep sweeping
            row = {"cfg": cfg, "error": str(exc)[:200]}
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
