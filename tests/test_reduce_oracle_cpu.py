"""The NumPy restatement of the fixed-order column reduction (oracle/reduce_oracle.py): its row
partition covers every row once with the part count csrc/reduce.cuh states, it is exact on
integer data, and its order is not the trivially order-free one."""
import numpy as np
import pytest

from oracle import reduce_oracle as ro


def sampled_sizes():
    edges = set()
    for p in range(1, ro.MAX_PARTS + 2):
        for d in (-1, 0, 1):
            edges.add(p * 1024 + d)
    edges.update(range(1, 2100))
    edges.update(np.unique(np.geomspace(1, 3_000_000, 2000).astype(int)).tolist())
    edges.update({8 * 1024 - 1, 8 * 1024 + 1, 10**6 + 3, 3_000_000, 2**24 + 3})
    return sorted(e for e in edges if e >= 1)


def test_partition_covers_every_row_once():
    for n in sampled_sizes():
        used, chunk = ro.row_parts(n)
        assert used == min(ro.ceil_div(n, 1024), 264), n
        assert chunk >= 1 and (used - 1) * chunk < n <= used * chunk, n
        # parts [p chunk, min(n, (p + 1) chunk)) tile [0, n): none empty, none overlapping
        starts = np.arange(used) * chunk
        ends = np.minimum(n, starts + chunk)
        assert np.all(ends > starts) and ends[-1] == n and np.all(starts[1:] == ends[:-1]), n


@pytest.mark.parametrize("n,used,chunk", [(1, 1, 1), (1024, 1, 1024), (1025, 2, 513),
                                          (8 * 1024 + 1, 9, 911), (264 * 1024, 264, 1024),
                                          (263 * 1024 + 1, 264, 1021), (264 * 1024 + 1, 264, 1025),
                                          (10**6 + 3, 264, 3788)])
def test_partition_examples(n, used, chunk):
    """Chunks are below 1024 rows whenever ceil(n / 1024) does not divide n evenly, and above it
    only past 264 * 1024 rows."""
    assert ro.row_parts(n) == (used, chunk)


@pytest.mark.parametrize("n", [1, 7, 8, 9, 1023, 1025, 1087, 8 * 1024 + 1, 263 * 1024 + 1, 300007])
def test_integer_data_is_exact(n):
    rng = np.random.default_rng(n)
    X = rng.integers(-(2**20), 2**20, size=(n, 5))
    np.testing.assert_array_equal(ro.column_sums(X.astype(np.float64)), X.sum(axis=0))


def test_order_matters_and_is_restated():
    """One large term per warp position and many small ones: the restated order rounds the small
    terms differently from a pairwise or sequential sum, and a single-part sum by hand agrees."""
    n = 3000
    rng = np.random.default_rng(1)
    X = rng.uniform(-1, 1, size=(n, 8)).astype(np.float32).astype(np.float64)
    X[::97] *= 2.0**40
    got = ro.column_sums(X)
    assert not np.array_equal(got, X.sum(axis=0))
    seq = np.zeros(8)
    for r in range(n):
        seq = seq + X[r]
    assert not np.array_equal(got, seq)
    # the same order spelled out row by row
    used, chunk = ro.row_parts(n)
    tot = np.zeros(8)
    for p in range(used):
        part = np.zeros(8)
        for w in range(8):
            acc = np.zeros(8)
            for r in range(p * chunk + w, min(n, (p + 1) * chunk), 8):
                acc = acc + X[r]
            part = part + acc
        tot = tot + part
    np.testing.assert_array_equal(got, tot)


def test_zero_padding_keeps_signed_zero_rules():
    """All-negative-zero columns sum to +0.0, as 0.0 + (-0.0) does on the device."""
    X = np.full((1025, 2), -0.0)
    got = ro.column_sums(X)
    assert np.all(got == 0) and not np.any(np.signbit(got))
