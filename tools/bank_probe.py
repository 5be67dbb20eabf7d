"""Times analysis and synthesis of wide filter banks on one GPU, old route against new.

    python tools/bank_probe.py [--n 1000000] [--nsig 64] [--order 30] [--reps 3]

On a 10-NN sensor graph (Morton order) with nsig signals and Chebyshev order 30, for
Nf in 2, 6, 16, 17, 64, 256, 2048 and float32 / float64:

  analysis   "fused": gsp_cheby_op_* (the fused step for 16 filters, then one read and write of
             every further accumulator per order; at most 1024 filters) against "basis": the
             stored basis and one combine pass (gsp_cheby_op_basis_*), for every Nf;
  synthesis  "loop": Nf forward recurrences summed (fused_synthesis=False) against "wide": the
             mix pass and one Clenshaw recurrence (gsp_cheby_synthesis_wide_*), and for Nf <= 16
             "clenshaw": the narrow fused synthesis of gsp_cheby_clenshaw_*.

Each line is JSON: times in ms (CUDA events, after a warm-up call), the largest difference
between the two routes relative to the largest output, and the passes over an (N, nsig) block
and the bytes the traffic model predicts (passes x N x nsig x itemsize; gathers, the matrix and
the coefficients are not counted):
  analysis fused  (m - 1)(2 Nf + 4)          basis  3 (m - 1) + m + Nf
  synthesis loop  Nf (5 (m - 1) + 3)         wide   Nf + m + 4 (m - 1)
A case whose buffers do not fit in the free device memory is reported as skipped.  The first line
names the card and its power limit.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
import pygsp_b200 as gsp  # noqa: E402
from pygsp_b200.filters import approximations as apx  # noqa: E402

NFS = (2, 6, 16, 17, 64, 256, 2048)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as exc:       # the name alone when nvidia-smi is not there
        return "%s (nvidia-smi: %s)" % (torch.cuda.get_device_name(), exc)


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        y = None               # one output alive at a time: the largest banks fill the card
        y = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps, y


def free_bytes():
    return apx._free_device_bytes(torch.device("cuda"))


def rel(a, b):
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-300))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--nsig", type=int, default=64)
    ap.add_argument("--order", type=int, default=30)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    m, nsig = args.order + 1, args.nsig
    print(json.dumps({"card": card(), "n": args.n, "nsig": nsig, "order": args.order}), flush=True)
    for dtype in (np.float32, np.float64):
        G = gsp.graphs.Sensor(args.n, k=10, seed=0, order="morton", dtype=dtype)
        G.estimate_lmax()
        L, n = G.L, G.N
        item = np.dtype(dtype).itemsize
        block = n * nsig * item
        rng = np.random.default_rng(0)
        x = torch.randn((n, nsig), dtype=L.dtype, device=L.device)
        for nf in NFS:
            c = rng.standard_normal((nf, m)) / np.arange(1, m + 1) ** 2
            base = {"dtype": np.dtype(dtype).name, "Nf": nf}
            # ------------------------------------------------------------------ analysis
            rec = dict(base, what="analysis",
                       model_bytes={"fused": (m - 1) * (2 * nf + 4) * block,
                                    "basis": (3 * (m - 1) + m + nf) * block})
            if (nf + m + 2) * block > 0.9 * free_bytes():
                rec["skipped"] = "needs %.1f GB" % ((nf + m + 2) * block / 2 ** 30)
            else:
                ms_b, yb = timed(lambda: apx.cheby_bank_device(L, G.lmax, c, x), args.reps)
                rec["ms"] = {"basis": ms_b}
                if nf <= 1024 and (2 * nf + 2) * block <= 0.9 * free_bytes():
                    ms_f, yf = timed(lambda: apx.cheby_op_device(L, G.lmax, c, x), args.reps)
                    rec["ms"]["fused"] = ms_f
                    rec["bit_identical"] = bool(torch.equal(yb, yf))
                    del yf
                del yb
            print(json.dumps(rec), flush=True)
            # ----------------------------------------------------------------- synthesis
            rec = dict(base, what="synthesis",
                       model_bytes={"loop": nf * (5 * (m - 1) + 3) * block,
                                    "wide": (nf + m + 4 * (m - 1)) * block})
            if (nf + m + 5) * block > 0.9 * free_bytes():
                rec["skipped"] = "needs %.1f GB" % ((nf + m + 5) * block / 2 ** 30)
                print(json.dumps(rec), flush=True)
                continue
            src = torch.randn((nf, n, nsig), dtype=L.dtype, device=L.device)

            def loop():
                out = torch.zeros((n, nsig), dtype=L.dtype, device=L.device)
                for i in range(nf):
                    out += apx.cheby_op_device(L, G.lmax, c[i], src[i])[0]
                return out

            ms_w, yw = timed(lambda: apx.cheby_synthesis_wide_device(L, G.lmax, c, src), args.reps)
            rec["ms"] = {"wide": ms_w}
            if nf <= 256:
                ms_l, yl = timed(loop, 1 if nf > 16 else args.reps)
                rec["ms"]["loop"] = ms_l
                rec["rel_diff_loop"] = rel(yw, yl)
            if nf <= 16:
                ms_c, yc = timed(lambda: apx.cheby_clenshaw_device(L, G.lmax, c, src), args.reps)
                rec["ms"]["clenshaw"] = ms_c
                rec["rel_diff_clenshaw"] = rel(yw, yc)
            print(json.dumps(rec), flush=True)
            del src
            torch.cuda.empty_cache()
        del G, L, x
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
