"""Per-stage timings of graph_multiresolution on the device (DESIGN.md section 4.11).

    python tools/multiresolution_probe.py [--n 10000] [--k 10] [--reps 3] [--out FILE]
                                          [--split eigenvector|random] [--keep 0.5]

Stages, each timed with CUDA events around device work that ends in a synchronise (median of
--reps runs after one warm-up):
  eigenvector   G._largest_eigenvector() (reflected ChFSI above 2048 vertices)
  kron_small    kron_reduction(L + 0.005 I, ind) at SMALL_MAX = s, for the s of --small
  resistances   the float64 factor of L + 11^T/N, its inverse, and the per-edge gather
  sampling      gsp_sparsify_sample for q = round(9 C^2 N log N / eps^2), eps = 0.3
and the removed-set statistics (components, largest) that set the small/dense threshold.
``--split random`` keeps each vertex with probability --keep (seeded) instead of the eigenvector
split, which on Morton k-NN graphs leaves one large removed component: a random split of a
sparser graph leaves many small ones, which is where the one-CTA kernel runs.  Prints one
JSON line with the card's name and power limit.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def timed(fn, reps):
    import torch
    fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        out.append(a.elapsed_time(b))
    return float(np.median(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10000)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--small", default="0,16,32,64,128")
    ap.add_argument("--out", default=None)
    ap.add_argument("--split", default="eigenvector", choices=["eigenvector", "random"])
    ap.add_argument("--keep", type=float, default=0.5)
    args = ap.parse_args()
    import torch
    import pygsp_b200 as gsp
    from pygsp_b200 import _native as nat
    from pygsp_b200 import reduction as red
    from pygsp_b200.graphs.csr import row_ids
    from scipy.sparse import csgraph

    G = gsp.graphs.Sensor(args.n, k=args.k, seed=1, order="morton", dtype=np.float64)
    res = {"n": args.n, "k": args.k, "nnz": G.W.nnz}
    res["eigenvector_ms"] = timed(lambda: G._largest_eigenvector(seed=0), args.reps)
    V = G._largest_eigenvector(seed=0)
    V *= np.sign(V[0])
    ind = np.nonzero(V >= 0)[0]
    if args.split == "random":
        ind = np.flatnonzero(np.random.default_rng(0).uniform(size=G.N) < args.keep)
    res["split"] = args.split
    L = G.L.to_scipy().astype(np.float64)
    rem = np.setdiff1d(np.arange(G.N), ind)
    nc, lab = csgraph.connected_components(L[rem][:, rem], directed=False)
    sizes = np.bincount(lab)
    res.update(kept=int(ind.size), components=int(nc), largest=int(sizes.max()))
    M = L + 0.005 * __import__("scipy").sparse.eye(G.N)
    ref = None
    for s in [int(v) for v in args.small.split(",")]:
        red.SMALL_MAX = s
        res["kron_small%d_ms" % s] = timed(lambda: red.kron_reduction(M, ind), args.reps)
        K = red.kron_reduction(M, ind)
        ref = K if ref is None else ref
        res["kron_small%d_maxdiff" % s] = float(abs(K - ref).max())
    res["kron_nnz"] = int(ref.nnz)

    Ld = red._device_matrix(G.L, G.device)

    def resist():
        rows, cols = row_ids(Ld.indptr), Ld.indices.long()
        e = rows > cols
        er, ec = rows[e].to(torch.int32).contiguous(), cols[e].to(torch.int32).contiguous()
        A, _, _ = red._laplacian_inverse(Ld)
        R = torch.empty(er.numel(), dtype=torch.float64, device=G.device)
        red._call("gsp_edge_resistance_f64", nat.i64(er.numel()), er, ec, A, nat.i64(G.N), R)
        return R
    res["resistances_ms"] = timed(resist, args.reps)
    R = resist()
    w = torch.ones_like(R)
    k = torch.round(w * R / (w * R).max() * 2.0 ** 32).to(torch.int64).contiguous()
    q = int(round(G.N * np.log(G.N) * 9 * (4 / 30.0) ** 2 / 0.3 ** 2))
    counts = torch.empty_like(k)
    res["q"] = q
    res["sampling_ms"] = timed(lambda: red._call("gsp_sparsify_sample", nat.i64(k.numel()), k,
                                                 nat.i64(q), nat.u64(1), counts), args.reps)
    try:
        res["gpu"] = subprocess.run(
            ["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as exc:   # pragma: no cover
        res["gpu"] = "unknown (%s)" % exc
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "a") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
