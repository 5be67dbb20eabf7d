"""Timing of graph_sparsify with exact and sketched effective resistances (needs a GPU).

    python tools/sparsify_probe.py [--reps 3] [--sizes 10000,100000,1000000] [--out FILE]

One JSON line per measurement (also appended to --out when given):
  card   : GPU name, power limit and SM clock limit (nvidia-smi), read in the same run;
  exact  : graph_sparsify(G, 0.3, resistances='exact') at N = 10^4 (the dense factor);
  sketch : graph_sparsify(G, 0.3, resistances='sketch') at every size, split into
           sketch_ms     -- the right-hand sides (gsp_jl_sketch_f64, all blocks),
           cg_ms         -- the block CG solves (learning._block_cg), with cg_iters per block,
           accumulate_ms -- the per-edge sums (gsp_jl_accumulate_f64, all blocks),
           sample_ms     -- the sampler (gsp_sparsify_sample, every epsilon attempt),
           other_ms      -- the rest: the float64 copy of L, edge lists, connectivity, the Graph.
G is Sensor(N, k=10, seed=1, order='morton') in float32, as a user builds it.  Times are
milliseconds, the median of --reps calls after one warm-up call; sizes of 10^6 and more are called
once, after the warm-up of the smaller sizes, since one call takes minutes.  Every part is timed by
a host clock around work that ends in a device synchronise (the probe synchronises around each
part, which the library itself does not).
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


class Split:
    """Times the parts of one graph_sparsify call by wrapping the reduction module's entry-point
    caller and the block CG driver."""
    PARTS = {"gsp_jl_sketch_f64": "sketch_ms", "gsp_jl_accumulate_f64": "accumulate_ms",
             "gsp_sparsify_sample": "sample_ms"}

    def __init__(self, reduction, learning, torch):
        self.red, self.lrn, self.torch = reduction, learning, torch
        self.call0, self.cg0 = reduction._call, learning._block_cg

    def timed(self, key, fn, *args):
        self.torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn(*args)
        self.torch.cuda.synchronize()
        self.t[key] = self.t.get(key, 0.0) + 1e3 * (time.perf_counter() - t0)
        return out

    def __enter__(self):
        self.t, self.iters = {}, []

        def call(name, *args):
            if name in self.PARTS:
                return self.timed(self.PARTS[name], self.call0, name, *args)
            return self.call0(name, *args)

        def cg(*args):
            X, done, worst = self.timed("cg_ms", self.cg0, *args)
            self.iters.append(done)
            return X, done, worst
        self.red._call, self.lrn._block_cg = call, cg
        return self

    def __exit__(self, *exc):
        self.red._call, self.lrn._block_cg = self.call0, self.cg0


def run(gsp, torch, G, how, reps, split):
    def once():
        with split:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            gsp.reduction.graph_sparsify(G, 0.3, seed=1, resistances=how)
            torch.cuda.synchronize()
            total = 1e3 * (time.perf_counter() - t0)
        parts = dict(split.t, total_ms=total)
        parts["other_ms"] = total - sum(v for k, v in split.t.items())
        return parts, list(split.iters)

    if reps > 1:
        once()
    calls = [once() for _ in range(max(reps, 1))]
    keys = calls[0][0].keys()
    med = {k: round(statistics.median(c[0][k] for c in calls), 1) for k in keys}
    return med, calls[-1][1]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--sizes", default="10000,100000,1000000")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    import pygsp_b200 as gsp
    from pygsp_b200 import learning
    emit({"card": card()}, args.out)
    split = Split(gsp.reduction, learning, torch)
    for n in [int(s) for s in args.sizes.split(",")]:
        G = gsp.graphs.Sensor(n, k=10, seed=1, order="morton")
        reps = args.reps if n < 10 ** 6 else 1
        base = {"N": n, "nnz": int(G.W.nnz), "k": gsp.reduction._sketch_dim(n),
                "width": gsp.reduction._sketch_width(n, gsp.reduction._sketch_dim(n)),
                "reps": reps}
        if n <= 10 ** 4:
            med, _ = run(gsp, torch, G, "exact", reps, split)
            emit(dict(base, what="exact", **med), args.out)
        med, iters = run(gsp, torch, G, "sketch", reps, split)
        emit(dict(base, what="sketch", cg_iters=iters, **med), args.out)
        del G
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
