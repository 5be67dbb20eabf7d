"""Generate tests/golden/random_graphs.npz from the unmodified PyGSP 0.6.1 (CPU).

    PYGSP_REFERENCE=<PyGSP 0.6.1 source tree> python tests/golden/make_golden_random_graphs.py

The reference's random streams cannot be shared by the device samplers, so only statistics of
its own runs are stored (read by tests/test_random_graphs_cpu.py and _gpu.py):

  sbm_<c>_z, sbm_<c>_M, sbm_<c>_flags   the model of SBM case <c>: blocks, probabilities and
                                        (directed, self_loops)
  sbm_<c>_counts                        (S, k, k) stored entries of W between blocks a and b, one
                                        row per seed 0 .. S - 1 (stochasticblockmodel.py:61-165;
                                        ErdosRenyi for c = 'er')
  ba_<c>_params                         (N, m0, m) of BarabasiAlbert case <c>
  ba_<c>_hist                           degree histogram summed over seeds 0 .. S_ba - 1
                                        (barabasialbert.py:43-65)
  ba_<c>_nseeds                         S_ba
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("PYGSP_REFERENCE") or (sys.argv[1] if len(sys.argv) > 1 else None)
OUT = os.path.join(HERE, "random_graphs.npz")

SEEDS = 300
BA_SEEDS = 200
_SORTED = np.repeat([0, 1, 2], [15, 20, 25])
_SHUFFLED = np.random.default_rng(5).permutation(_SORTED)
# name: (z, M, directed, self_loops)
SBM = {
    "default": (_SORTED, None, False, False),
    "directed": (_SORTED, None, True, False),
    "loops": (_SORTED, None, False, True),
    "asym": (_SORTED, np.array([[0.3, 0.02, 0.1], [0.05, 0.2, 0.04], [0.2, 0.01, 0.25]]),
             False, False),
    "unsorted": (_SHUFFLED, None, False, False),
}
ER = (60, 0.1)
BA = {"n300_m1": (300, 1, 1), "n500_m2": (500, 3, 2), "n1000_m4": (1000, 4, 4)}


def default_M(k, p=0.3, q=0.05):
    M = np.full((k, k), q)
    M.flat[::k + 1] = p
    return M


def block_counts(W, z, k):
    coo = W.tocoo()
    C = np.zeros((k, k), dtype=np.int64)
    np.add.at(C, (z[coo.row], z[coo.col]), 1)
    return C


def main():
    if not REF:
        raise SystemExit("set PYGSP_REFERENCE to the PyGSP 0.6.1 source tree")
    sys.path.insert(0, REF)
    from pygsp import graphs

    out = {}
    for name, (z, M, directed, self_loops) in SBM.items():
        k = int(z.max()) + 1
        M = default_M(k) if M is None else M
        counts = []
        for seed in range(SEEDS):
            G = graphs.StochasticBlockModel(N=z.size, k=k, z=z, M=M.copy(), directed=directed,
                                            self_loops=self_loops, seed=seed)
            counts.append(block_counts(G.W, z, k))
        out["sbm_%s_z" % name] = z
        out["sbm_%s_M" % name] = M
        out["sbm_%s_flags" % name] = np.array([directed, self_loops])
        out["sbm_%s_counts" % name] = np.array(counts)
        print(name, np.mean(counts, axis=0).ravel())
    N, p = ER
    counts = [graphs.ErdosRenyi(N=N, p=p, seed=seed).W.nnz for seed in range(SEEDS)]
    out["sbm_er_z"] = np.zeros(N, dtype=np.int64)
    out["sbm_er_M"] = np.array([[p]])
    out["sbm_er_flags"] = np.array([False, False])
    out["sbm_er_counts"] = np.array(counts, dtype=np.int64).reshape(-1, 1, 1)
    for name, (N, m0, m) in BA.items():
        hist = np.zeros(N, dtype=np.int64)
        for seed in range(BA_SEEDS):
            deg = np.asarray((graphs.BarabasiAlbert(N=N, m0=m0, m=m, seed=seed).W > 0).sum(axis=1))
            hist += np.bincount(deg.ravel(), minlength=N)[:N]
        out["ba_%s_params" % name] = np.array([N, m0, m])
        out["ba_%s_hist" % name] = hist
        out["ba_%s_nseeds" % name] = np.array(BA_SEEDS)
        print(name, hist[:12])
    np.savez_compressed(OUT, **out)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
