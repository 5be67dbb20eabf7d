"""Generate tests/golden/random_regular.npz from the unmodified PyGSP 0.6.1 (CPU).

    PYGSP_REFERENCE=<PyGSP 0.6.1 source tree> python tests/golden/make_golden_random_regular.py

The reference's ``RandomRegular`` (randomregular.py) is run once per seed, each run in a worker
process under a timeout: its restart rebuilds the stub array as floats and then raises, and a run
that is stuck after more than N k tests never ends.  Its random stream cannot be shared by the
device sampler, so only statistics of its own runs are stored (read by
tests/test_random_regular_cpu.py):

  rr_<c>_params       (N, k, number of seeds S); seeds are 0 .. S - 1
  rr_<c>_outcome      (successes, errors, timeouts) over the S seeds
  rr_<c>_triangles    triangle count of every successful run (a k-regular graph), in seed order
  rr_<c>_lambda2      second smallest eigenvalue of its combinatorial Laplacian, same order
  rr_6_2_classes      at (6, 2): successful runs that gave the hexagon and two triangles
"""
import multiprocessing as mp
import os
import signal
import sys

os.environ.setdefault("OMP_NUM_THREADS", "1")     # one BLAS thread per worker process

import numpy as np
from scipy import sparse

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("PYGSP_REFERENCE") or (sys.argv[1] if len(sys.argv) > 1 else None)
OUT = os.path.join(HERE, "random_regular.npz")

# name: (N, k, seeds, timeout in seconds)
CASES = {"6_2": (6, 2, 4000, 2), "64_6": (64, 6, 400, 20), "200_20": (200, 20, 200, 30),
         "1000_6": (1000, 6, 200, 60), "2000_10": (2000, 10, 100, 120)}


class _Timeout(Exception):
    pass


def _alarm(signum, frame):
    raise _Timeout()


def _run(args):
    """(status, triangles, lambda2) of one reference run: status 0 ok, 1 error, 2 timeout or
    not k-regular."""
    N, k, seed, timeout = args
    import logging
    logging.disable(logging.WARNING)
    from pygsp import graphs
    signal.signal(signal.SIGALRM, _alarm)
    signal.alarm(timeout)
    try:
        G = graphs.RandomRegular(N=N, k=k, seed=seed)
    except _Timeout:
        return 2, -1, np.nan
    except Exception:                      # the reference's float-index restart
        signal.alarm(0)
        return 1, -1, np.nan
    signal.alarm(0)
    A = sparse.csr_matrix((G.W > 0).astype(np.float64))
    deg = np.asarray(A.sum(axis=0)).ravel()
    if not (deg == k).all():               # max_iter ran out
        return 2, -1, np.nan
    tri = int(round((A @ A).multiply(A).sum() / 6))
    L = (sparse.diags(deg) - A).toarray()
    lam2 = float(np.linalg.eigvalsh(L)[1])
    return 0, tri, lam2


def main():
    if not REF:
        raise SystemExit("set PYGSP_REFERENCE to the PyGSP 0.6.1 source tree")
    sys.path.insert(0, REF)
    os.environ["PYTHONPATH"] = REF + os.pathsep + os.environ.get("PYTHONPATH", "")
    out = {}
    with mp.get_context("fork").Pool(max(1, os.cpu_count() - 1), maxtasksperchild=50) as pool:
        for name, (N, k, S, timeout) in CASES.items():
            res = pool.map(_run, [(N, k, s, timeout) for s in range(S)], chunksize=1)
            status = np.array([r[0] for r in res])
            ok = status == 0
            tri = np.array([r[1] for r in res], dtype=np.int64)[ok]
            lam2 = np.array([r[2] for r in res], dtype=np.float64)[ok]
            out["rr_%s_params" % name] = np.array([N, k, S])
            out["rr_%s_outcome" % name] = np.array([(status == v).sum() for v in (0, 1, 2)])
            out["rr_%s_triangles" % name] = tri
            out["rr_%s_lambda2" % name] = lam2
            if name == "6_2":
                out["rr_6_2_classes"] = np.array([(tri == 0).sum(), (tri == 2).sum()])
            print(name, out["rr_%s_outcome" % name], tri.mean(), lam2.mean(), flush=True)
    np.savez_compressed(OUT, **out)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
