"""Timing of the spring layout (csrc/layout.cu) and of the reference's algorithm on the host.

    python tools/layout_probe.py [--iters 5] [--reference <PyGSP 0.6.1 tree>]

Per-iteration time of ``gsp_spring_step_*`` (CUDA events, median over --iters launches after one
warm-up) on Sensor(N, k=10, seed=0) graphs, N = 1e4, 1e5, 1e6, with and without
``order='morton'``, from a seeded uniform start.  The achieved rate is N^2 pairs per iteration
over the time; its share of the FP64 issue ceiling is

    pairs/s * (FP64 instructions per pair) / (132 SMs * 64 FP64 lanes * 1.98 GHz),

the instructions per pair read from the SASS of the dim = 2 kernel (cuobjdump): the FP64
instructions of its candidate loop over the MUFU.RCP64H instructions (one per pair) of that
loop.  The host rows time 50 iterations at N = 1000 and 2000 of the float64 NumPy restatement
of the reference's loop (oracle/layout_oracle.py) and, with --reference, of the unmodified
reference itself.  The card's name and power limit are printed with the numbers.  One JSON line
per case.
"""
import argparse
import json
import os
import re
import shutil
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

FP64_PEAK = 132 * 64 * 1.98e9          # H100 SXM: FP64 lanes x boost clock, instructions/s
FP64_OPS = ("DADD", "DMUL", "DFMA", "DSETP", "DMNMX")


def sass_dp_per_pair():
    """FP64 instructions per pair of the dim = 2 repulsion kernel, from its SASS (None if
    cuobjdump is not available)."""
    from pygsp_b200 import build
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool):
        return None
    sass = subprocess.run([tool, "-sass", build.LIB], capture_output=True, text=True).stdout
    for fn in re.split(r"\n\s*Function : ", sass)[1:]:
        if "spring_repulsion_kernelILi2E" not in fn.split("\n")[0]:
            continue
        lines = [ln for ln in fn.split("\n") if re.search(r"/\*[0-9a-f]{4}\*/", ln)]
        addr = [int(re.search(r"/\*([0-9a-f]{4})\*/", ln).group(1), 16) for ln in lines]
        best = None            # innermost backward-branch loop that computes pairs
        for i, ln in enumerate(lines):
            m = re.search(r"BRA (0x[0-9a-f]+)", ln)
            if not m or int(m.group(1), 16) >= addr[i]:
                continue
            body = lines[addr.index(int(m.group(1), 16)):i + 1]
            ops = [re.search(r"\*/\s+(?:@!?U?P\w+\s+)?([A-Z0-9_.]+)", ln).group(1) for ln in body]
            mufu = sum(op == "MUFU.RCP64H" for op in ops)
            if mufu and (best is None or len(body) < best[0]):
                dp = sum(op.split(".")[0] in FP64_OPS for op in ops)
                best = (len(body), dp / mufu)
        return None if best is None else best[1]
    return None


def card():
    import torch
    out = {"gpu": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        out["power_limit_and_max_sm_clock"] = q.stdout.strip().splitlines()[0]
    except Exception as exc:          # the numbers are still printed, the limit is "not measured"
        out["power_limit_and_max_sm_clock"] = "not measured (%s)" % type(exc).__name__
    return out


def device_rows(args, dp):
    import torch

    import pygsp_b200 as gsp
    from pygsp_b200 import _native as nat
    for n in (10 ** 4, 10 ** 5, 10 ** 6):
        for order in (None, "morton"):
            G = gsp.graphs.Sensor(n, k=10, seed=0, order=order)
            W = G.W
            cur = torch.as_tensor(np.random.default_rng(0).uniform(size=(n, 2)), device=G.device)
            nxt = torch.empty_like(cur)
            k = float(np.sqrt(1.0 / n))

            def step():
                G._call("gsp_spring_step", nat.i64(n), nat.i32(2), W.indptr, W.indices, W.data,
                        nat.f64(k), nat.f64(0.1), None, cur, nxt)
            step()
            torch.cuda.synchronize()
            times = []
            for _ in range(args.iters):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                step()
                b.record()
                torch.cuda.synchronize()
                times.append(a.elapsed_time(b) * 1e-3)
            sec = float(np.median(times))
            pairs = float(n) * float(n) / sec
            row = {"case": "device_step", "n": n, "order": order, "dim": 2,
                   "iteration_s": sec, "iteration_s_min": float(min(times)),
                   "pairs_per_s": pairs, "fp64_per_pair_sass": dp,
                   "fp64_issue_share": None if dp is None else pairs * dp / FP64_PEAK,
                   "layout_50_iterations_s": 50 * sec}
            print(json.dumps(row), flush=True)
            del G, cur, nxt
            torch.cuda.empty_cache()


def host_rows(args):
    from scipy import sparse

    from oracle import layout_oracle as lo
    for n in (1000, 2000):
        rng = np.random.default_rng(n)
        W = sparse.random(n, n, density=10.0 / n, random_state=rng)
        W = sparse.csr_matrix(sparse.triu(W, 1) + sparse.triu(W, 1).T)
        t0 = time.perf_counter()
        lo.run(W, 2, None, None, [], 50, 0)
        row = {"case": "host_numpy_restatement", "n": n, "iterations": 50,
               "seconds": time.perf_counter() - t0, "host_cpus": len(os.sched_getaffinity(0))}
        if args.reference:
            sys.path.insert(0, args.reference)
            from pygsp.graphs import _layout
            t0 = time.perf_counter()
            _layout._sparse_fruchterman_reingold(W > 0, 2, None, None, [], 50, 0)
            row["reference_seconds"] = time.perf_counter() - t0
        print(json.dumps(row), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--reference", default=None, help="PyGSP 0.6.1 source tree (host rows)")
    ap.add_argument("--host-only", action="store_true")
    args = ap.parse_args()
    if not args.host_only:
        import torch
        if not torch.cuda.is_available():
            raise SystemExit("layout_probe: no CUDA device (use --host-only for the host rows)")
        dp = sass_dp_per_pair()
        print(json.dumps({"case": "card", **card(), "fp64_per_pair_sass": dp}), flush=True)
        device_rows(args, dp)
    host_rows(args)


if __name__ == "__main__":
    main()
