"""The serial restatement of the exact-size subset sampler (oracle/sampled_models_oracle.py):
exact counts, distinct pairs inside their spaces, and uniform subset frequencies over a fixed
set of keys (deterministic chi-square tests).  No GPU needed."""
import itertools
from collections import Counter

import numpy as np
import pytest
from scipy import stats

from oracle import sampled_models_oracle as smo

RECT, TRI = smo.RECT, smo.TRI_STRICT


def _pairs(rows, cols):
    """Unordered pairs of the (u, v), (v, u) entries."""
    assert np.array_equal(rows[0::2], cols[1::2]) and np.array_equal(cols[0::2], rows[1::2])
    return [(int(u), int(v)) for u, v in zip(rows[0::2], cols[0::2])]


def _two_communities():
    """Communities {0, 1} and {2, 3, 4}: two intra triangles and the 3 x 2 rectangle."""
    return [([(TRI, 1, 2, 0, 0)], 1), ([(TRI, 3, 3, 2, 2)], 2), ([(RECT, 6, 2, 2, 0)], 3)]


@pytest.mark.parametrize("key", [1, 2 ** 40 + 7, 2 ** 63 - 5])
def test_exact_counts_and_distinct_pairs(key):
    spaces = [([(TRI, 45, 10, 0, 0)], 17), ([(TRI, 190, 20, 10, 10)], 0),
              ([(RECT, 200, 10, 10, 0)], 200), ([(RECT, 200, 10, 30, 0), (RECT, 300, 20, 50, 10)],
                                                 11)]
    rows, cols, _ = smo.subset_pairs(80, spaces, key)
    pairs = _pairs(rows, cols)
    assert len(pairs) == 17 + 200 + 11
    assert len(set(pairs)) == len(pairs)
    first = pairs[:17]
    assert all(10 > u > v >= 0 for u, v in first)
    assert sorted(pairs[17:217]) == sorted((10 + i, j) for i in range(20) for j in range(10))
    assert all((30 <= u < 50 and v < 10) or (50 <= u < 65 and 10 <= v < 30)
               for u, v in pairs[217:])


def _chi2(counts, n_outcomes):
    obs = np.array([counts.get(k, 0) for k in sorted(counts)] +
                   [0] * (n_outcomes - len(counts)))
    return stats.chisquare(obs).pvalue


def test_uniform_subsets_of_a_small_space():
    """M = 6, n = 2: all 15 subsets equally likely over 3000 fixed keys."""
    counts = Counter()
    for key in range(3000):
        rows, cols, _ = smo.subset_pairs(4, [([(TRI, 6, 4, 0, 0)], 2)], key * 7919 + 1)
        counts[frozenset(_pairs(rows, cols))] += 1
    assert len(counts) == 15
    assert _chi2(counts, 15) > 1e-4


def test_uniform_subsets_of_two_communities():
    """Sizes 2 and 3: every space's subset uniform, spaces independent."""
    per_space = [Counter(), Counter(), Counter()]
    joint = Counter()
    for key in range(3000):
        rows, cols, _ = smo.subset_pairs(5, _two_communities(), 104729 * key + 3)
        pairs = _pairs(rows, cols)
        parts = (frozenset(pairs[:1]), frozenset(pairs[1:3]), frozenset(pairs[3:]))
        for c, part in zip(per_space, parts):
            c[part] += 1
        joint[(parts[1], parts[2])] += 1
    assert len(per_space[0]) == 1
    assert len(per_space[1]) == 3 and _chi2(per_space[1], 3) > 1e-4
    assert len(per_space[2]) == 20 and _chi2(per_space[2], 20) > 1e-4
    table = np.zeros((3, 20))
    a = {k: i for i, k in enumerate(sorted(per_space[1], key=sorted))}
    b = {k: i for i, k in enumerate(sorted(per_space[2], key=sorted))}
    for (x, y), c in joint.items():
        table[a[x], b[y]] = c
    assert stats.chi2_contingency(table).pvalue > 1e-4


def test_full_and_empty_targets():
    rows, cols, _ = smo.subset_pairs(4, [([(TRI, 6, 4, 0, 0)], 6)], 11)
    assert sorted(_pairs(rows, cols)) == sorted((j, i) for i, j in
                                                itertools.combinations(range(4), 2))
    rows, cols, _ = smo.subset_pairs(4, [([(TRI, 6, 4, 0, 0)], 0)], 11)
    assert rows.size == 0
