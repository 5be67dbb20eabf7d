"""Timing of the structured-graph kernels and the line graph (needs a GPU).

    python tools/structured_probe.py [--reps 10] [--out FILE]

One JSON line per measurement (also appended to --out when given):
  card       : GPU name, power limit and SM clock limit (nvidia-smi), read in the same run;
  line_graph : the line graph of the config-2 graph (Sensor-type k-NN, 1e6 vertices, k = 10,
               Morton order, float32): gsp_line_graph_count and gsp_line_graph_fill separately,
               and LineGraph(G) end to end (D, edge list, count, fill and the Graph checks);
  torus      : gsp_torus_count of Torus(10_000, 10_000) alone (row sizes, int64 total, scan), and
               the whole adjacency (count, fill);
  full       : the adjacency of FullConnected(30_000) (indptr, fill).
Times are milliseconds per call from CUDA events after warm-up calls.  Each is reported beside
the time the bytes it stores would take at the H100 SXM data-sheet HBM bandwidth (3.35 TB/s):
4 bytes per row pointer, 4 + 4 per float32 entry.  That bound is a model, not a measurement.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_PEAK = 3.35e12          # H100 SXM data sheet


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


def timed(fn, reps, warmup=2):
    import torch
    for _ in range(warmup):
        fn()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(reps):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / reps


def record(kind, ms, stored, out, **extra):
    emit(dict(kind=kind, ms=round(ms, 4), stored_bytes=int(stored),
              write_bound_ms=round(stored / HBM_PEAK * 1e3, 4),
              share_of_write_bound=round(stored / HBM_PEAK * 1e3 / ms, 3), **extra), out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("structured_probe needs a CUDA device")
    import pygsp_b200 as gsp
    from pygsp_b200 import _native as nat
    from pygsp_b200.graphs.csr import DeviceCSR
    emit(dict(kind="card", card=card(), torch=torch.__version__), a.out)

    # ---- line graph of config 2: count and fill apart
    G = gsp.graphs.Sensor(1_000_000, k=10, seed=0, order="morton")
    G.compute_differential_operator()
    D, W, ne, dev = G.D, G.W, G.n_edges, G.device
    _, s, t, _, _ = G._edges_device()
    lg_indptr = torch.empty(ne + 1, dtype=torch.int32, device=dev)
    nnz = torch.empty(1, dtype=torch.int64, device=dev)
    st = nat.stream_ptr(dev)
    head = (nat.i64(ne), s, t, D.indptr)
    tail = (W.indptr, W.indices, nat.i32(0), lg_indptr)

    def count():
        nat.call("gsp_line_graph_count", *head, *tail, nnz, st)
    ms = timed(count, a.reps)
    total = int(nnz.item())
    record("line_graph_count", ms, 4 * (ne + 1), a.out, n_edges=ne, nnz=total)
    indices = torch.empty(total, dtype=torch.int32, device=dev)
    data = torch.empty(total, dtype=torch.float32, device=dev)

    def fill():
        nat.call("gsp_line_graph_fill_f32", *head, D.indices, *tail, indices, data, st)
    ms = timed(fill, a.reps)
    record("line_graph_fill", ms, 8 * total, a.out, n_edges=ne, nnz=total)
    del indices, data
    ms = timed(lambda: gsp.graphs.LineGraph(G), max(2, a.reps // 5), warmup=1)
    record("LineGraph", ms, 4 * (ne + 1) + 8 * total, a.out, n_edges=ne, nnz=total)
    del G, D, W, s, t

    # ---- Torus(10_000, 10_000) and FullConnected(30_000) adjacencies
    args = (nat.i64(10_000), nat.i64(10_000))
    indptr = torch.empty(10 ** 8 + 1, dtype=torch.int32, device=dev)

    def torus_count():
        nat.call("gsp_torus_count", *args, indptr, nnz, st)
    ms = timed(torus_count, a.reps)
    record("torus_count", ms, 4 * (10 ** 8 + 1), a.out, n=10 ** 8, nnz=int(nnz.item()))
    del indptr

    def torus():
        return DeviceCSR.from_counts(
            (10 ** 8, 10 ** 8), torch.float32, dev,
            lambda st, ip, total: nat.call("gsp_torus_count", *args, ip, total, st),
            lambda st, ip, ix, d: nat.call("gsp_torus_fill_f32", *args, ip, ix, d, st), "graph")
    ms = timed(torus, a.reps)
    record("torus", ms, 4 * (10 ** 8 + 1) + 8 * 4 * 10 ** 8, a.out, n=10 ** 8, nnz=4 * 10 ** 8)

    n = 30_000

    def full():
        return DeviceCSR.from_counts(
            (n, n), torch.float32, dev,
            lambda st, ip, total: nat.call("gsp_full_connected_indptr", nat.i64(n), ip, total, st),
            lambda st, ip, ix, d: nat.call("gsp_full_connected_fill_f32", nat.i64(n), ix, d, st),
            "graph")
    ms = timed(full, a.reps)
    record("full", ms, 4 * (n + 1) + 8 * n * (n - 1), a.out, n=n, nnz=n * (n - 1))


if __name__ == "__main__":
    main()
