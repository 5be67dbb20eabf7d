"""Generate tests/golden/dropin.npz from the unmodified PyGSP 0.6.1 (CPU, SciPy path).

    PYGSP_REFERENCE=<PyGSP 0.6.1 source tree> python tests/golden/make_golden_dropin.py

Two parts, both read by tests/test_reference_dropin_gpu.py:
  objects: the README's Logo example through stock pygsp objects -- Heat(50).filter on three
           deltas, MexicanHat(Nf=5) analysis of a block at order 40 and analysis + synthesis
           at order 25 -- with the reference's own lmax draw.  The block is 7 columns of
           default_rng(0); columns are filtered independently, so only the first column is
           stored, and the results only at OBJ_ROWS rows drawn with default_rng(1) ("obj_rows");
  suite  : every cheby_op call that the reference's own pygsp/tests/test_filters.py makes
           (Laplacian, lmax, coefficients, signal and SciPy result of each), recorded while
           that test file runs unmodified.  Repeated calls (same graph, lmax, coefficients and
           signal) count once; SUITE_CALLS of the distinct calls, drawn with default_rng(0), are
           stored.  Coefficient and signal arrays that several stored calls share are stored
           once ("suite_pool_<i>").  Calls on graphs larger than 200 vertices or with more than
           64 signal columns are not recorded (none at present).
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("PYGSP_REFERENCE") or (sys.argv[1] if len(sys.argv) > 1 else None)
OUT = os.path.join(HERE, "dropin.npz")
OBJ_ROWS = 256
SUITE_CALLS = 24


class Recorder:
    """pytest plugin: wraps pygsp.filters.approximations.cheby_op and keeps every call."""

    def __init__(self):
        self.calls, self.laplacians = [], []

    def pytest_configure(self, config):
        import pygsp.filters.approximations as apx
        stock = apx.cheby_op

        def recorded(G, c, signal, **kw):
            out = stock(G, c, signal, **kw)
            L = G.L.tocsr()
            if G.N <= 200 and np.ndim(signal) <= 2 and np.size(signal) <= 64 * G.N:
                for gi, known in enumerate(self.laplacians):
                    if known.shape == L.shape and (known != L).nnz == 0:
                        break
                else:
                    gi = len(self.laplacians)
                    self.laplacians.append(L.copy())
                self.calls.append((gi, float(G.lmax), np.array(c, dtype=np.float64),
                                   np.array(signal, dtype=np.float64),
                                   np.array(out, dtype=np.float64)))
            return out
        apx.cheby_op = recorded


def objects(pygsp):
    G = pygsp.graphs.Logo()
    G.estimate_lmax()
    s = np.zeros(G.N)
    s[[20, 30, 1090]] = 1
    bank = pygsp.filters.MexicanHat(G, Nf=5)
    heat = pygsp.filters.Heat(G, scale=50)
    block = np.random.default_rng(0).standard_normal((G.N, 7))
    rows = np.sort(np.random.default_rng(1).choice(G.N, size=OBJ_ROWS, replace=False))
    return {"obj_lmax": np.float64(G.lmax), "obj_deltas": s, "obj_block": block[:, :1],
            "obj_rows": rows.astype(np.int64),
            "obj_heat": heat.filter(s)[rows],
            "obj_bank_o40": bank.filter(block, order=40)[rows, :1],
            "obj_bank_bank_o25": bank.filter(bank.filter(block), order=25)[rows, :1]}


def main():
    if not REF:
        raise SystemExit(__doc__)
    sys.path.insert(0, REF)
    import logging
    import pytest
    import pygsp
    logging.getLogger("pygsp").setLevel(logging.ERROR)
    out = objects(pygsp)
    rec = Recorder()
    rc = pytest.main(["-q", "-p", "no:cacheprovider",
                      os.path.join(REF, "pygsp", "tests", "test_filters.py")], plugins=[rec])
    assert rc == 0, rc
    for gi, L in enumerate(rec.laplacians):
        L = L.tocsr()
        L.sort_indices()
        out["suite_L%d_indptr" % gi] = L.indptr.astype(np.int64)
        out["suite_L%d_indices" % gi] = L.indices.astype(np.int64)
        out["suite_L%d_data" % gi] = L.data
        out["suite_L%d_shape" % gi] = np.array(L.shape, dtype=np.int64)
    pool = {}

    def pooled(a):
        key = (a.shape, a.tobytes())
        if key not in pool:
            pool[key] = len(pool)
            out["suite_pool_%d" % pool[key]] = a
        return pool[key]
    distinct = {}
    for call in rec.calls:
        gi, lmax, c, x, _ = call
        distinct.setdefault((gi, lmax, c.shape, c.tobytes(), x.shape, x.tobytes()), call)
    distinct = list(distinct.values())
    keep = np.random.default_rng(0).choice(len(distinct), size=min(SUITE_CALLS, len(distinct)),
                                           replace=False)
    for i, j in enumerate(sorted(keep)):
        gi, lmax, c, x, y = distinct[j]
        out["suite_%03d_ids" % i] = np.array([gi, pooled(c), pooled(x)], dtype=np.int64)
        out["suite_%03d_lmax" % i] = np.float64(lmax)
        out["suite_%03d_y" % i] = y
    out["suite_calls"] = np.int64(len(keep))
    np.savez_compressed(OUT, **out)
    print("%s: %d of %d distinct suite calls (%d in all) on %d graphs, %d bytes"
          % (OUT, len(keep), len(distinct), len(rec.calls), len(rec.laplacians),
             os.path.getsize(OUT)))


if __name__ == "__main__":
    main()
