"""Random regular graphs on the host: the serial restatement of the device sampler
(oracle/random_regular_oracle.py) against the exact law of the reference's sequential rule, over
every small case, and against statistics of the reference's own runs
(tests/golden/random_regular.npz); the input errors, which are raised before the device is used."""
import os
import re

import numpy as np
import pytest
from scipy import sparse
from scipy.sparse.linalg import eigsh

from conftest import ROOT, load_golden
from oracle import random_regular_oracle as rro


def _key(seed):
    return int(np.random.default_rng(seed).integers(2 ** 63))


def test_constants_match_header():
    """The oracle and the Python module restate the determinism constants of the header."""
    from pygsp_b200.graphs import random_graphs
    text = open(os.path.join(ROOT, "include", "gspb200.h")).read()

    def macro(name):
        m = re.search(r"#define GSPB200_RR_%s \(?([0-9xA-Fa-f]+)(?:ull)?(?: << (\d+)\))?" % name,
                      text)
        assert m, name
        v = int(m.group(1), 0)
        return v << int(m.group(2)) if m.group(2) else v
    assert macro("TAIL_STUBS") == rro.TAIL_STUBS == random_graphs._TAIL_STUBS
    assert macro("CHECK_AFTER") == rro.CHECK_AFTER
    assert macro("TAIL_DRAWS") == rro.TAIL_DRAWS
    assert macro("SWITCH_DRAWS") == rro.SWITCH_DRAWS
    assert macro("MAX_ROUNDS") == rro.MAX_ROUNDS
    assert macro("TAIL_STREAM") == rro.TAIL_STREAM
    assert macro("SWITCH_STREAM") == rro.SWITCH_STREAM


@pytest.mark.parametrize("N,k", [(5, 2), (6, 2), (7, 2), (8, 2), (8, 3)])
def test_serial_law_matches_reference_rule(N, k):
    """Graph-class frequencies of the restatement over 20 000 keys, default max_iter, against the
    exact law of the reference's rule conditioned on success: within 4 standard errors per class."""
    law = rro.exact_law(N, k)
    assert abs(sum(law.values()) - 1) < 1e-12
    S = 20000
    seen, counts = {}, dict.fromkeys(law, 0)
    for key in np.random.default_rng(100 * N + k).integers(2 ** 63, size=S).tolist():
        eu, ev, _, _, complete = rro.random_regular_edges(N, k, 10, key)
        assert complete
        g = frozenset(zip(np.minimum(eu, ev).tolist(), np.maximum(eu, ev).tolist()))
        if g not in seen:
            seen[g] = rro.graph_class(N, g)
        counts[seen[g]] += 1
    for c, p in law.items():
        assert abs(counts[c] / S - p) <= 4 * np.sqrt(p * (1 - p) / S), (c, counts[c] / S, p)


def test_exact_law_matches_reference_runs():
    """The reference's own (6, 2) runs: two triangles as often as the exact law says."""
    g = load_golden("random_regular")
    hexagon, triangles = (int(v) for v in g["rr_6_2_classes"])
    n = hexagon + triangles
    p = [v for c, v in rro.exact_law(6, 2).items() if min(c) > -1.5]
    assert len(p) == 1                  # two triangles: spectrum (-1)^4 2^2; the hexagon's has -2
    p = p[0]
    assert abs(triangles / n - p) <= 4 * np.sqrt(p * (1 - p) / n)


def _simple_regular(N, k, eu, ev):
    u, v = np.array(eu, dtype=np.int64), np.array(ev, dtype=np.int64)
    if (u == v).any():
        return False
    ck = np.minimum(u, v) * N + np.maximum(u, v)
    deg = np.bincount(np.concatenate([u, v]), minlength=N)
    return np.unique(ck).size == ck.size and (deg == k).all()


def test_every_small_case_is_regular():
    """Every N <= 16, 0 <= k <= N - 1 with N k even, seeds 0..99, default max_iter: the graph is
    k-regular, simple and symmetric (the complement included)."""
    for N in range(1, 17):
        for k in range(N):
            if N * k % 2:
                continue
            kk = N - 1 - k if 2 * k > N - 1 else k
            for seed in range(100):
                eu, ev, _, _, complete = rro.random_regular_edges(N, kk, 10, _key(seed))
                assert complete and _simple_regular(N, kk, eu, ev), (N, k, seed)
    for N, k in ((7, 4), (10, 9), (16, 9), (16, 15)):
        W, _, _ = rro.random_regular_graph(N, k, 10, _key(3))
        assert (W != W.T).nnz == 0 and W.diagonal().sum() == 0
        assert set(W.data) == {1.0} and (np.diff(W.indptr) == k).all()


def _triangles_lambda2(W):
    A = W.astype(np.float64)
    tri = int(round((A @ A).multiply(A).sum() / 6))
    L = (sparse.diags(np.asarray(A.sum(axis=1)).ravel()) - A).tocsc()
    lam = np.sort(eigsh(L, k=2, sigma=-0.01, which="LM", return_eigenvectors=False))
    return tri, float(lam[1])


@pytest.mark.parametrize("case,seeds", [("64_6", 300), ("1000_6", 60), ("2000_10", 40)])
def test_statistics_match_reference(case, seeds):
    """Triangle count and lambda_2 means of the restatement against the reference's runs: within
    4 combined standard errors.  (1000, 6) and (2000, 10) take the pairing rounds first."""
    g = load_golden("random_regular")
    N, k, _ = (int(v) for v in g["rr_%s_params" % case])
    ours = np.array([_triangles_lambda2(rro.random_regular_graph(N, k, 10, _key(10 ** 4 + s))[0])
                     for s in range(seeds)])
    if N * k > rro.TAIL_STUBS:
        assert rro.random_regular_graph(N, k, 10, _key(10 ** 4))[2] >= 1
    for col, ref in ((0, g["rr_%s_triangles" % case]), (1, g["rr_%s_lambda2" % case])):
        se = np.sqrt(ours[:, col].var() / len(ours) + ref.var() / len(ref))
        assert abs(ours[:, col].mean() - ref.mean()) <= 4 * max(se, 1e-12), (col, ours[:, col].mean(),
                                                                              ref.mean())


def test_input_errors_are_raised_before_the_device():
    from pygsp_b200 import graphs
    with pytest.raises(ValueError, match=r"input error: N\*d must be even!"):
        graphs.RandomRegular(N=7, k=3)
    with pytest.raises(ValueError, match="non-negative"):
        graphs.RandomRegular(N=8, k=-2)
    for N, k in ((6, 6), (6, 8), (1, 2)):
        with pytest.raises(ValueError, match="does not exist"):
            graphs.RandomRegular(N=N, k=k)
    with pytest.raises(ValueError, match="max_iter"):
        graphs.RandomRegular(N=8, k=2, max_iter=0)
    with pytest.raises(ValueError, match="at most 2"):
        graphs.RandomRegular(N=2 ** 28, k=8)
