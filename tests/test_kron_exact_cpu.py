"""Host restatements behind tests/test_kron_exact_gpu.py (oracle/kron_exact_oracle.py): the builder
of matrices with prescribed removed components, the component structure the device must reproduce,
and the replay of every draw of gsp_sparsify_sample against a plain per-draw loop."""
import numpy as np
import pytest
from scipy import sparse
from scipy.sparse import csgraph

from oracle import kron_exact_oracle as keo
from oracle.random_graphs_oracle import philox4x32_10

SPECS = {
    "edges": [(1, 1, "well"), (1, 2, "well"), (2, 1, "well"), (2, 1, "ill"), (17, 9, "ill"),
              (18, 9, "well"), (3, 0, "well")],
    "budget": [(64, 126, "well"), (8, 300, "ill"), (64, 127, "ill"), (65, 10, "well")],
    "status": [(6, 5, "well")] * 10 + [(5, 4, "indefinite")] + [(9, 7, "ill")] * 10,
}


def _kept_neighbours(M, v, kept_index):
    cols = np.unique(M[v].indices)
    k = kept_index[cols]
    return np.sort(k[k >= 0])


@pytest.mark.parametrize("name", sorted(SPECS))
@pytest.mark.parametrize("seed", [0, 1])
def test_builder_makes_the_requested_components(name, seed):
    specs = SPECS[name]
    M, ind, comps = keo.build_components(specs, seed=seed)
    n, m = M.shape[0], ind.size
    assert abs(M - M.T).max() == 0
    assert np.unique(ind).size == m
    kept_index = np.full(n, -1)
    kept_index[ind] = np.arange(m)
    rem = np.flatnonzero(kept_index < 0)
    assert rem.size == sum(s for s, _, _ in specs)
    # kept and removed ids interleave, and so does the kept order
    assert rem.min() < ind.max() and ind.min() < rem.max()
    assert not np.all(np.diff(ind) > 0)

    nc, lab = csgraph.connected_components(M[rem][:, rem], directed=False)
    assert nc == len(specs)
    firsts = []
    for c, ((s, b, kind), comp) in enumerate(zip(specs, comps)):
        v = comp["vertices"]
        assert v.size == s and comp["s"] == s and comp["b"] == b and comp["kind"] == kind
        labels = lab[np.searchsorted(rem, v)]
        assert np.all(labels == labels[0])
        assert np.count_nonzero(lab == labels[0]) == s          # exactly this component
        firsts.append(v.min())
        kept = _kept_neighbours(M, v, kept_index)
        assert kept.size == b
        np.testing.assert_array_equal(kept, comp["kept"])
        A = M[v][:, v].toarray()
        ev = np.linalg.eigvalsh(A)
        kappa = np.linalg.cond(A)
        if kind == "well":
            assert ev.min() > 0 and kappa <= 100
        elif kind == "ill":
            assert ev.min() > 0
            assert kappa >= (1e7 if s >= 16 else 1e6 if s >= 8 else 1.0)
        else:
            assert ev.min() < 0 and np.all(np.diag(A) > 0)
    assert np.all(np.diff(firsts) > 0)              # specs in order of their smallest vertex
    # the kept neighbours of different components interleave in kept-index order
    spans = [(c["kept"].min(), c["kept"].max()) for c in comps if c["b"] >= 2]
    assert any(a0 < b1 and b0 < a1 for i, (a0, a1) in enumerate(spans)
               for (b0, b1) in spans[i + 1:])


@pytest.mark.parametrize("name", sorted(SPECS))
def test_removed_components_match_the_builder(name):
    M, ind, comps = keo.build_components(SPECS[name], seed=3)
    got = keo.removed_components(M, ind)
    assert len(got) == len(comps)
    for g, c in zip(got, comps):
        np.testing.assert_array_equal(g["vertices"], c["vertices"])
        np.testing.assert_array_equal(g["kept"], c["kept"])


def test_schur_blocks_against_the_dense_schur_complement():
    """The per-component blocks summed into M[ind, ind] give the dense Schur complement."""
    from oracle import multiresolution_oracle as mro
    M, ind, _ = keo.build_components(SPECS["edges"] + [(30, 12, "well"), (40, 15, "ill")],
                                     seed=4)
    blocks = keo.schur_blocks(M, ind)
    K = M[ind][:, ind].toarray()
    for blk in blocks:
        K[np.ix_(blk["kept"], blk["kept"])] += blk["block"]
    want = mro.kron_matrix(M, ind)
    tol = keo.schur_tolerance(M, ind, blocks)
    assert np.all(np.abs(K - want) <= tol)


def _counts_loop(k, q, seed):
    """gsp_sparsify_sample draw by draw in plain Python integers."""
    mask = 0xFFFFFFFF
    cum, acc = [], 0
    for v in k:
        acc += int(v)
        cum.append(acc)
    total = cum[-1]
    counts = [0] * len(k)
    for d in range(q):
        chunk, off = d // 128, d % 128
        t = off // 2
        x, y, z, w = philox4x32_10((t & mask, t >> 32, chunk & mask, chunk >> 32),
                                   (seed & mask, seed >> 32))
        r = (x << 32 | y) if off % 2 == 0 else (z << 32 | w)
        u = r * total >> 64
        e = 0
        while not cum[e] > u:
            e += 1
        counts[e] += 1
    return np.array(counts, dtype=np.int64)


def _weights(name):
    rng = np.random.default_rng(7)
    if name == "random":
        return rng.integers(0, 1000, 50)
    if name == "zeros":
        k = rng.integers(1, 40, 60)
        k[0] = k[-1] = 0
        k[10:17] = 0
        k[30] = 0
        return k
    if name == "one_edge":
        return np.array([5])
    if name == "near_2^63":
        k = [int(v) for v in rng.integers(2 ** 59, 2 ** 60, 7)]
        return np.array(k + [2 ** 63 - 1 - sum(k)], dtype=np.uint64)
    return np.array({"ones": [1, 1, 1], "gap": [1, 0, 2], "single3": [3]}[name])


@pytest.mark.parametrize("name", ["random", "zeros", "one_edge", "near_2^63", "ones", "gap",
                                  "single3"])
def test_sparsify_replay_matches_the_per_draw_loop(name):
    k = _weights(name)
    for q, seed in ((0, 1), (1, 2), (2, 3), (127, 4), (128, 5), (129, 6), (300, 2 ** 64 - 1)):
        got = keo.sparsify_counts(k, q, seed)
        np.testing.assert_array_equal(got, _counts_loop(k, q, seed))
        assert got.sum() == q
        assert np.all(got[np.asarray(k) == 0] == 0)
