"""The random-walk Schur complement of kron_reduction(method='walks'), restated in NumPy
(oracle/schur_walks_oracle.py): unbiased against the dense Schur complement, the closed form of a
three-vertex path, the cases that need no sampling, and the spectrum of a sampled k-NN level."""
import numpy as np
import pytest
from scipy import sparse

from oracle import schur_walks_oracle as swo


def _path(weights):
    n = len(weights) + 1
    W = sparse.diags([weights, weights], [-1, 1], shape=(n, n))
    return (sparse.diags(np.asarray(W.sum(axis=1)).ravel()) - W).tocsr()


def _grid3(reg=0.0):
    rows, cols = [], []
    for i in range(3):
        for j in range(3):
            v = 3 * i + j
            if j < 2:
                rows.append(v), cols.append(v + 1)
            if i < 2:
                rows.append(v), cols.append(v + 3)
    w = np.array([1.0, 2.0, 0.5, 1.5, 3.0, 1.0, 0.25, 2.0, 1.0, 1.0, 4.0, 0.75])
    W = sparse.coo_matrix((w, (rows, cols)), shape=(9, 9))
    W = (W + W.T).tocsr()
    return (sparse.diags(np.asarray(W.sum(axis=1)).ravel() + reg) - W).tocsr()


def _replicates(M, ind, samples, key):
    """(samples, m, m) array: replicate r is the exact part plus every item r mod samples, each at
    its unscaled weight -- one full sample of the Laplacian."""
    m = len(ind)
    res = swo.walk_items(M, ind, samples, key)
    out = np.zeros((samples, m, m))
    r0, c0, v0 = swo.exact_part(M, ind)
    np.add.at(out, (slice(None), r0, c0), v0)
    c1, c2 = res["c1"], res["c2"]
    live = (c1 != c2) & (c1 != swo.CAPPED) & (c2 != swo.CAPPED)
    rep = res["item"] % samples
    val = res["val"] * samples
    for i in np.flatnonzero(live):
        a, b = c1[i], c2[i]
        if a == swo.GROUND or b == swo.GROUND:
            k = b if a == swo.GROUND else a
            out[rep[i], k, k] += val[i]
        else:
            out[rep[i], a, b] -= val[i]
            out[rep[i], b, a] -= val[i]
            out[rep[i], a, a] += val[i]
            out[rep[i], b, b] += val[i]
    return out


@pytest.mark.parametrize("case", ["path6", "grid3", "grid3_reg"])
def test_unbiased(case):
    M, ind = {"path6": (_path([1.0, 2.0, 0.5, 3.0, 1.5]), [0, 5]),
              "grid3": (_grid3(), [0, 2, 6, 8]),
              "grid3_reg": (_grid3(0.05), [0, 2, 6, 8])}[case]
    samples = 20_000
    Y = _replicates(M, np.array(ind), samples, key=0xC0FFEE + len(case))
    mean = Y.mean(axis=0)
    se = Y.std(axis=0, ddof=1) / np.sqrt(samples)
    SC = swo.dense_schur(M, ind)
    scale = np.abs(SC).max()
    assert np.all(np.abs(mean - SC) <= 5 * se + 1e-12 * scale), (mean - SC) / np.maximum(se, 1e-300)
    # the oracle's own reduction is that mean
    H = swo.schur_walks(M, ind, samples, key=0xC0FFEE + len(case)).toarray()
    np.testing.assert_allclose(H, mean, rtol=0, atol=1e-12 * scale)


def test_three_vertex_path_closed_form():
    w1, w2 = 2.0, 3.0
    M = _path([w1, w2])
    samples = 40_000
    res = swo.walk_items(M, [0, 2], samples, key=7)
    edge0 = res["item"] < samples                     # the edge (1, 0) of weight w1
    sample = np.where(res["c1"] != res["c2"], res["val"] * samples, 0.0)
    target = 1.0 / (1.0 / w1 + 1.0 / w2)
    nz = sample != 0
    np.testing.assert_allclose(sample[nz], target, rtol=1e-15)
    p = w2 / (w1 + w2)
    freq = nz[edge0].mean()
    assert abs(freq - p) <= 5 * np.sqrt(p * (1 - p) / samples)
    assert set(np.unique(res["steps"])) == {1}


def test_nothing_removed_is_exact():
    M = _grid3(0.05)
    ind = np.array([4, 0, 8, 1, 7, 2, 6, 3, 5])
    H = swo.schur_walks(M, ind, 16, key=1)
    assert (H != M[ind][:, ind]).nnz == 0
    np.testing.assert_array_equal(H.diagonal(), M.diagonal()[ind])


def test_components_without_kept_neighbours_add_nothing():
    A = _grid3()
    B = _path([1.0, 2.0, 3.0])                      # removed entirely: no kept neighbour
    M = sparse.block_diag([A, B]).tocsr()
    ind = np.array([0, 2, 6, 8])
    eu, ev, _, gu = swo.items(M, ind)
    assert eu.max() < 9 and ev.max() < 9 and gu.size == 0
    _, dead = swo.split(M, ind)
    np.testing.assert_array_equal(np.flatnonzero(dead), np.arange(9, 13))
    H1 = swo.schur_walks(M, ind, 8, key=3)
    H2 = swo.schur_walks(A, ind, 8, key=3)
    assert (H1 != H2).nnz == 0


def test_kept_excess_is_exact():
    """A kept vertex's excess is its own exact sample: removing nothing around it leaves it."""
    M = sparse.block_diag([_grid3(), sparse.csr_matrix([[2.5]])]).tocsr()
    H = swo.schur_walks(M, [0, 2, 6, 8, 9], 4, key=5).toarray()
    assert H[4, 4] == 2.5 and not H[4, :4].any()


def test_prep_flags_and_cap():
    M = _path([1.0, 1.0]).tolil()
    M[0, 1] = M[1, 0] = 0.5
    assert swo.prep(M.tocsr())[3] & 1
    M = _path([1.0, 1.0]).tolil()
    M[1, 1] = 1.5
    assert swo.prep(M.tocsr())[3] & 2
    P = _path(np.ones(49))
    res = swo.walk_items(P, [0, 49], 1, key=0, max_steps=10)
    assert (res["c1"] == swo.CAPPED).any() or (res["c2"] == swo.CAPPED).any()
    assert res["steps"].max() <= 10


def test_spectrum_of_a_knn_level():
    """The 2-D k-NN case of DESIGN.md section 4.23 at N = 1500 with 16 samples per edge."""
    L = swo.knn_laplacian(1500, k=10, seed=0)
    ind = swo.eigenvector_split(L)
    SC = swo.dense_schur(L, ind)
    res = swo.walk_items(L, ind, 16, key=11)
    H = swo.schur_walks(L, ind, 16, key=11).toarray()
    lo, hi = swo.generalized_spread(H, SC)
    print("N = 1500, 16 samples: spread [%.3f, %.3f], fro %.3f, entries %d / %d, steps mean %.2f "
          "max %d" % (lo, hi, np.linalg.norm(H - SC) / np.linalg.norm(SC), np.count_nonzero(H),
                      np.count_nonzero(np.abs(SC) > 1e-12 * np.abs(SC).max()),
                      res["steps"].mean(), res["steps"].max()))
    assert 0.8 <= lo and hi <= 1.25
