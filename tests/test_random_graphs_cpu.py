"""Random graph models on the host: the Philox restatement, the decoders and chunk plan, the
laws of the serial restatements, and the host SBM sampler (no GPU needed)."""
import hashlib

import numpy as np
import pytest
from scipy import stats

from conftest import load_golden
from oracle import random_graphs_oracle as rgo


def test_philox_known_answers():
    """Random123's known-answer vectors for Philox4x32-10 (kat_vectors)."""
    kat = [((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
           ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
           ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
            (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]
    for ctr, key, want in kat:
        assert rgo.philox4x32_10(ctr, key) == want
        got = rgo.philox4x32_10(tuple(np.array([c], dtype=np.uint64) for c in ctr),
                                tuple(np.uint64(k) for k in key))
        assert tuple(int(w[0]) for w in got) == want


@pytest.mark.parametrize("kind,n,width", [(0, 1, 1), (0, 35, 7), (1, 1, 2), (1, 4950, 100),
                                          (2, 1, 1), (2, 5050, 100), (3, 2, 2), (3, 9900, 100)])
def test_decoders_are_bijections(kind, n, width):
    from pygsp_b200.graphs.random_graphs import decode_pairs, pair_space
    i, j = decode_pairs(kind, np.arange(n), width)
    pairs = list(zip(i.tolist(), j.tolist()))
    assert len(set(pairs)) == n
    assert pairs == [rgo.decode(kind, x, width) for x in range(n)]
    if kind == 0 and n == 35:
        want = {(a, b) for a in range(5) for b in range(7)}
        assert pair_space(5, 7, False, False, False) == (0, 35, 7)
    else:
        directed, loops = kind in (0, 3), kind in (0, 2)
        assert pair_space(width, width, True, directed, loops) == (kind, n, width)
        want = {(a, b) for a in range(width) for b in range(width)
                if (directed or b <= a) and (loops or a != b)}
    assert set(pairs) == want


def test_decoders_exact_at_large_indices():
    """The square root is corrected in integers where float64 rounding would be off."""
    from pygsp_b200.graphs.random_graphs import decode_pairs
    for kind, s in ((1, 1), (2, -1)):
        i = np.array([10 ** 7, 3 * 10 ** 7 + 17, 94906266], dtype=np.int64)
        for off in (0, 1):
            idx = i * (i - s) // 2 + (i - 1 if kind == 1 else i) * off
            di, dj = decode_pairs(kind, idx, 0)
            assert np.array_equal(di, i) and np.array_equal(dj, (i - 1 if kind == 1 else i) * off)


@pytest.mark.parametrize("target", [1e-9, 1.0, 64, 1e12])
def test_chunk_plan_covers_every_index_once(target):
    from pygsp_b200.graphs.random_graphs import sbm_plan
    M = np.array([[1.0, 0.3, 0.0], [0.3, 0.02, 0.5], [0.0, 0.5, 0.7]])
    for directed in (False, True):
        for loops in (False, True):
            plan, prob, n_chunks = sbm_plan(np.array([3, 7, 1]), M, directed, loops, target)
            ref = rgo.chunk_plan([3, 7, 1], M, directed, loops, target)
            assert len(plan) == len(ref) and n_chunks == sum(b["nch"] for b in ref)
            assert np.array_equal(plan[:, 2], np.cumsum([0] + [b["nch"] for b in ref])[:-1])
            for row, pr, b in zip(plan, prob, ref):
                n, clen, cfirst, r0, c0, width, kind, mirror = row.tolist()
                assert (n, clen, kind, width, r0, c0) == (b["n"], b["clen"], b["kind"], b["width"],
                                                         b["row0"], b["col0"])
                assert mirror == int(not directed) and pr[0] == b["p"]
                nch = -(-n // clen)
                cover = np.concatenate([np.arange(c * clen, min(c * clen + clen, n))
                                        for c in range(nch)])
                assert np.array_equal(cover, np.arange(n))
                if target <= 1e-9:
                    assert clen == 1
                if target >= 1e12:
                    assert clen == n


def test_serial_sbm_inclusion_and_independence_across_chunks():
    """ErdosRenyi(12, p) with one expected edge per chunk (chunks of 4 indices): every pair's
    frequency and the joint frequency of index pairs straddling a chunk boundary are binomial."""
    N, p, S = 12, 0.3, 2000
    M = np.array([[p]])
    n = N * (N - 1) // 2
    hits = np.zeros((S, n), dtype=bool)
    for s in range(S):
        for blk in rgo.chunk_plan([N], M, False, False, target=1.0):
            assert blk["clen"] == 4
            hits[s, rgo.walk(blk, 1000 + s)] = True
    freq = hits.mean(axis=0)
    sd = np.sqrt(p * (1 - p) / S)
    assert np.abs(freq - p).max() < 4.5 * sd
    b = np.arange(4, n, 4)
    joint = (hits[:, b - 1] & hits[:, b]).mean(axis=0)
    sdj = np.sqrt(p * p * (1 - p * p) / S)
    assert np.abs(joint - p * p).max() < 4.5 * sdj
    inside = (hits[:, b - 2] & hits[:, b - 1]).mean(axis=0)
    assert np.abs(inside - p * p).max() < 4.5 * sdj


@pytest.mark.parametrize("N,m0,m", [(5, 1, 1), (6, 2, 2), (6, 3, 2)])
def test_serial_ba_matches_exact_law(N, m0, m):
    law = rgo.ba_exact_law(N, m0, m)
    assert abs(sum(law.values()) - 1) < 1e-12
    graphs = sorted(law, key=sorted)
    index = {g: t for t, g in enumerate(graphs)}
    S = 3000
    obs = np.zeros(len(graphs))
    for s in range(S):
        t = rgo.ba_targets(N, m0, m, 7 * s + 1)
        i = m0 + np.arange(len(t)) // m
        obs[index[frozenset(zip(t, i.tolist()))]] += 1
    expected = S * np.array([law[g] for g in graphs])
    assert stats.chisquare(obs, expected).pvalue > 1e-4


def _hash(W):
    W = W.tocsr()
    return hashlib.sha256(np.ascontiguousarray(W.indptr, np.int64).tobytes()
                          + np.ascontiguousarray(W.indices, np.int64).tobytes()
                          + np.ascontiguousarray(W.data, np.float64).tobytes()).hexdigest()[:16]


def test_host_sbm_default_draws_unchanged():
    """Hashes of W recorded before the directed / self-loop pair spaces were added."""
    from pygsp_b200.graphs.generators import sbm_adjacency
    cases = [(dict(N=200, k=3, seed=0), 12006, "af2352cf9d48544c"),
             (dict(N=200, k=3, seed=1), 11862, "b13b5894fa04a598"),
             (dict(N=1000, k=5, p=0.1, q=0.01, seed=7), 28060, "f5ecfc745fb19aba"),
             (dict(N=500, k=4, p=[0.2, 0.3, 0.4, 0.5], q=0.05, seed=3), 31136, "ccfd687211946fd8")]
    for args, nnz, h in cases:
        W, _ = sbm_adjacency(**args)
        assert W.nnz == nnz and _hash(W) == h


def block_zscores(counts, z, M, directed, self_loops):
    """z-scores of per-block-pair stored-entry counts (S, k, k) against the model's binomial law."""
    k = M.shape[0]
    sizes = np.bincount(z, minlength=k).astype(float)
    pairs = np.outer(sizes, sizes)
    if not self_loops:
        pairs.flat[::k + 1] -= sizes
    P = M.copy() if directed else np.tril(M) + np.tril(M, -1).T
    mean = pairs * P
    var = pairs * P * (1 - P)
    if not directed:          # an edge inside a block is stored twice, a loop once
        dP = np.diag(P)
        var.flat[::k + 1] = 2 * np.diag(var) - (sizes * dP * (1 - dP) if self_loops else 0)
    return (counts - mean) / np.sqrt(np.maximum(var, 1e-9))


def host_counts(name, g, seeds):
    from pygsp_b200.graphs.generators import _sbm_draw
    z, M = g["sbm_%s_z" % name], g["sbm_%s_M" % name]
    directed, loops = (bool(f) for f in g["sbm_%s_flags" % name])
    k = M.shape[0]
    out = []
    for s in seeds:
        W = _sbm_draw(np.random.default_rng(s), z.size, k, z, M, directed, loops)
        assert set(np.unique(W.data)) <= {1.0}
        if not loops:
            assert W.diagonal().sum() == 0
        if not directed:
            assert (W != W.T).nnz == 0
        coo = W.tocoo()
        C = np.zeros((k, k), dtype=np.int64)
        np.add.at(C, (z[coo.row], z[coo.col]), 1)
        out.append(C)
    return np.array(out)


def compare_to_golden(ours, ref):
    """Per-block-pair means of two samples of counts agree within a Welch bound."""
    m1, m2 = ours.mean(0), ref.mean(0)
    se = np.sqrt(ours.var(0) / len(ours) + ref.var(0) / len(ref))
    return np.abs(m1 - m2) / np.maximum(se, 1e-9)


@pytest.mark.parametrize("name", ["directed", "loops", "asym"])
def test_host_sbm_variants_match_reference(name):
    g = load_golden("random_graphs")
    ours = host_counts(name, g, range(300))
    assert compare_to_golden(ours, g["sbm_%s_counts" % name]).max() < 4.5
    z = g["sbm_%s_z" % name]
    directed, loops = (bool(f) for f in g["sbm_%s_flags" % name])
    zs = block_zscores(ours, z, g["sbm_%s_M" % name], directed, loops)
    assert abs(zs.mean()) < 0.2 and 0.8 < zs.std() < 1.2
