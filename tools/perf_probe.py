"""Interleaved A/B timing of the recurrence forms on the bench workload (needs a GPU).

    python tools/perf_probe.py [--n 1000000] [--rounds 5] [--calls 10]

Builds BASELINE config 2 once and times, round-robin in ONE process (so that machine state,
allocator state and clocks are shared): forward recurrence, Clenshaw form, and the same with
GSPB200_* toggles flipped at run time (the library reads them per launch).  One JSON line per
variant with every round's ms per call.
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
    ap.add_argument("--order", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("variants", nargs="*",
                    default=["forward", "clenshaw", "clenshaw:TILE_REV=0", "forward:TILE_REV=0",
                             "clenshaw:TILE_HINT=0"])
    a = ap.parse_args()
    import torch
    import bench
    import pygsp_b200 as gsp
    from pygsp_b200.filters import approximations as apx

    G = gsp.graphs.Sensor(a.n, k=a.k, seed=0, order="morton")
    G.estimate_lmax()
    g = gsp.filters.Heat(G, scale=50)
    c = np.atleast_2d(gsp.filters.compute_cheby_coeff(g, m=a.order))
    x = torch.randn(G.N, a.nsig, device="cuda", generator=torch.Generator("cuda").manual_seed(0))
    out = torch.empty((1, G.N, a.nsig), device="cuda")
    work = torch.empty((2, G.N, a.nsig), device="cuda")
    peak, _ = bench.measured_peak()

    def run(form):
        if form == "forward":
            apx.cheby_op_device(G.L, G.lmax, c, x, out=out, work=work)
        else:
            apx.cheby_clenshaw_device(G.L, G.lmax, c, x, out=out[0], work=work)

    results = {v: [] for v in a.variants}
    reference, equal = {}, {}
    for rnd in range(a.rounds + 1):                     # round 0 = warm-up
        for v in a.variants:
            form, _, env = v.partition(":")
            sets = dict(kv.split("=") for kv in env.split(",") if kv)
            for k, val in sets.items():
                os.environ["GSPB200_" + k] = val
            G.L._plans.clear()                        # the tiling reads the toggles too
            run(form)
            torch.cuda.synchronize()
            if rnd == 0:                              # every variant must give the form's bits
                got = (out[0] if form != "forward" else out).clone()
                equal[v] = bool(torch.equal(got, reference.setdefault(form, got)))
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for _ in range(a.calls):
                run(form)
            e.record()
            torch.cuda.synchronize()
            for k in sets:
                del os.environ["GSPB200_" + k]
            if rnd:
                results[v].append(s.elapsed_time(e) / a.calls)
    for v, ms in results.items():
        form = v.partition(":")[0]
        _, _, b = bench.algorithmic_bytes(G.N, G.L.nnz, a.nsig, 1, a.order, clenshaw=form != "forward")
        best = min(ms)
        print(json.dumps({"variant": v, "ms_per_call_rounds": [round(t, 3) for t in ms],
                          "bit_identical_to_first_variant_of_form": equal.get(v),
                          "best_ms": round(best, 3), "frac_best": round(b / best / 1e6 / peak, 3),
                          "units_per_s_best": G.N * a.nsig * a.order / best * 1e3}), flush=True)


if __name__ == "__main__":
    main()
