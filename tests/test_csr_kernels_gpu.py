"""The sparse-structure kernels every Graph passes through, against SciPy / NumPy at the shapes
where row-per-thread, count -> scan -> fill and radix-key code breaks.

Covered: COO assembly (``gsp_coo_to_csr_*``), transpose, the five symmetrisations, zero
compaction, induced submatrices (``gsp_vertex_map`` / ``gsp_subgraph_*``), ``gsp_csr_inspect_*``,
asymmetry, weighted degree, the two Laplacians, the spectral bounds, row gather / scatter and
the SpMV / SpMM on heavy and empty rows.  Each one is held to the exactness it promises: values
that are only moved are compared bit for bit, sums whose order is fixed are compared bit for bit
with the same order on the host, and only ``pow`` and FMA contraction get a tolerance.

The matrix zoo holds empty matrices and rows (the last row included), n = 1, a star whose centre
row and column hold more than 2^16 entries, a directed matrix with one-sided, mirrored-unequal,
cancelling, negative, stored-zero and -0.0 entries and loops, loop-only vertices, and vertex counts
at and just past powers of two with entries in the highest rows and columns (the radix keys take
their width from n).  All values are float32 numbers, so one matrix serves both dtypes.
"""
import functools

import numpy as np
import pytest
from scipy import sparse

from oracle import nngraph_oracle as nno
from oracle import pygsp_oracle as orc

pytestmark = pytest.mark.gpu

DTYPES = [np.float32, np.float64]
METHODS = ["average", "maximum", "fill", "tril", "triu"]


@pytest.fixture(scope="module")
def gsp():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import pygsp_b200
    return pygsp_b200


# ------------------------------------------------------------------------------- the zoo
def _csr(n, r, c, v):
    """n x n CSR holding exactly the entries (r, c, v), stored zeros included; of two entries at
    one position the first is kept.  Values are rounded to float32 and stored as float64."""
    r, c = np.asarray(r, np.int64), np.asarray(c, np.int64)
    v = np.asarray(v, np.float64).astype(np.float32).astype(np.float64)
    key, first = np.unique(r * n + c, return_index=True)
    r, c, v = (key // n, key % n, v[first]) if n else (r, c, v)
    indptr = np.concatenate([[0], np.cumsum(np.bincount(r, minlength=n))]).astype(np.int32)
    return sparse.csr_matrix((v, c.astype(np.int32), indptr), shape=(n, n))


def _sym(n, r, c, v):
    """Undirected: both (r, c) and (c, r) with the same value (the first one given for a pair)."""
    r, c = np.asarray(r, np.int64), np.asarray(c, np.int64)
    _, first = np.unique(np.minimum(r, c) * n + np.maximum(r, c), return_index=True)
    r, c, v = r[first], c[first], np.asarray(v)[first]
    return _csr(n, np.concatenate([r, c]), np.concatenate([c, r]), np.concatenate([v, v]))


def _directed(rng):
    n = 300
    pairs = set()
    while len(pairs) < 560:
        i, j = sorted(rng.integers(0, n, 2))
        if i != j:
            pairs.add((int(i), int(j)))
    pairs = np.array(sorted(pairs))
    rng.shuffle(pairs)
    i, j = pairs[:, 0], pairs[:, 1]
    w = rng.uniform(0.1, 2.0, len(i)) * np.where(rng.random(len(i)) < 0.2, -1.0, 1.0)
    w2 = rng.uniform(0.1, 2.0, len(i))
    r, c, v = [], [], []

    def add(rr, cc, vv):
        r.append(rr); c.append(cc); v.append(vv)
    add(i[:100], j[:100], w[:100]); add(j[:100], i[:100], w[:100])                # mirrored, equal
    add(i[100:200], j[100:200], w[100:200]); add(j[100:200], i[100:200], w2[100:200])  # unequal
    add(i[200:300], j[200:300], w[200:300])                                        # one-sided
    add(j[300:400], i[300:400], w[300:400])                                        # one-sided
    add(i[400:410], j[400:410], -w2[400:410]); add(j[400:410], i[400:410], w2[400:410])  # cancel
    add(i[410:420], j[410:420], np.zeros(10)); add(j[410:420], i[410:420], w[410:420])  # 0 / w
    add(i[420:430], j[420:430], np.full(10, -0.0))                                 # lone -0.0
    add(i[430:440], j[430:440], np.full(10, -0.0)); add(j[430:440], i[430:440], np.zeros(10))
    add(i[440:450], j[440:450], np.zeros(10))                                      # lone 0
    add(i[450:560], j[450:560], -w[450:560]); add(j[450:560], i[450:560], -w[450:560])  # negative
    loops = rng.choice(n, 20, replace=False)
    add(loops, loops, rng.uniform(-1.0, 3.0, 20))
    add([5], [5], [0.0])                                                           # stored 0 loop
    return _csr(n, np.concatenate(r), np.concatenate(c), np.concatenate(v))


def _high(n, rng, directed):
    """Entries in the highest-numbered rows and columns, a few reaching down to 0 and n/2."""
    top = np.arange(n - 48, n)
    i, j = rng.choice(top, 200), rng.choice(top, 200)
    keep = i != j
    i, j = np.concatenate([i[keep], [n - 1, n - 1, n - 2]]), np.concatenate([j[keep], [0, n // 2, 1]])
    w = rng.uniform(0.1, 4.0, len(i))
    M = _sym(n, i, j, w)
    loop = _csr(n, [n - 1], [n - 1], [1.25])
    if directed:
        M = M + _csr(n, [n - 3, n - 1, 0], [n - 1, 2, n - 5], [0.5, 3.0, 7.0])
    return (M + loop).tocsr()


def _build(name):
    rng = np.random.default_rng(sum(map(ord, name)))
    if name == "n0":
        return _csr(0, [], [], [])
    if name == "n1":
        return _csr(1, [], [], [])
    if name == "n1_loop":
        return _csr(1, [0], [0], [2.5])
    if name == "n1000_nnz0":
        return _csr(1000, [], [], [])
    if name == "path":
        n = 64
        return _sym(n, np.arange(n - 1), np.arange(1, n), rng.uniform(0.5, 2.0, n - 1))
    if name == "star":
        n = 70_001                        # row 0 and column 0 hold 70 000 > 2^16 entries
        w = rng.uniform(0.1, 1.0, n - 1) * 10.0 ** rng.uniform(-3, 3, n - 1)
        return _sym(n, np.zeros(n - 1, np.int64), np.arange(1, n), w)
    if name == "directed":
        return _directed(rng)
    if name == "isolated":
        n = 41                            # odd vertices and the last one (40) have no entry
        ev = np.arange(0, 39, 2)
        return _sym(n, ev[:-1], ev[1:], rng.uniform(0.5, 2.0, len(ev) - 1))
    if name == "loop_only":
        n = 6                             # vertices 3 and 4: the loop is their only entry
        M = _sym(n, [0, 1, 2], [1, 2, 5], [1.0, 2.0, 0.5])
        return (M + _csr(n, [3, 4], [3, 4], [1.5, 4.0])).tocsr()
    if name == "n65536":
        return _high(2 ** 16, rng, directed=False)
    if name == "n65537":
        return _high(2 ** 16 + 1, rng, directed=True)
    if name == "n1048579":
        return _high(2 ** 20 + 3, rng, directed=True)
    raise KeyError(name)


CASES = ["n0", "n1", "n1_loop", "n1000_nnz0", "path", "star", "directed", "isolated", "loop_only",
         "n65536", "n65537", "n1048579"]


@functools.lru_cache(maxsize=None)
def zoo(name):
    M = _build(name).tocsr()
    M.data = M.data.astype(np.float32).astype(np.float64)     # sums of _high's overlapping parts
    assert M.has_sorted_indices and M.dtype == np.float64
    return M


def host(M, dtype):
    """M with its values in dtype (exact: the zoo's values are float32 numbers)."""
    return M.astype(dtype)


def canonical64(M, dtype):
    """What Graph keeps of M in dtype, as float64: the stored zeros (and -0.0) removed."""
    W = M.astype(dtype).astype(np.float64)
    W.eliminate_zeros()
    return W


def bits(a):
    a = np.ascontiguousarray(a)
    return a.view({4: np.uint32, 8: np.uint64}[a.dtype.itemsize])


def tdtype(dtype):
    import torch
    return torch.float32 if dtype == np.float32 else torch.float64


def device(gsp, M, dtype):
    import torch
    return gsp.graphs.DeviceCSR.from_scipy(M, tdtype(dtype), torch.device("cuda"))


def assert_csr_bits(D, ref, dtype):
    """DeviceCSR D == SciPy ref: indptr, indices and the bits of the values in dtype."""
    ref = ref.tocsr()
    assert D.shape == ref.shape
    np.testing.assert_array_equal(D.indptr.cpu().numpy(), ref.indptr)
    np.testing.assert_array_equal(D.indices.cpu().numpy(), ref.indices)
    np.testing.assert_array_equal(bits(D.data.cpu().numpy()), bits(ref.data.astype(dtype)))


def seq_row_sums(M):
    """Row sums of M in float64, each accumulated from 0 in stored order (no pairwise summation)."""
    M = M.tocsr()
    n = M.shape[0]
    lens = np.diff(M.indptr)
    order = np.argsort(-lens, kind="stable")
    sl, start = lens[order], M.indptr[:-1][order]
    data = M.data.astype(np.float64)
    acc = np.zeros(n)
    for k in range(int(sl[0]) if n else 0):
        m = int(np.searchsorted(-sl, -k, side="left"))     # rows longer than k
        acc[:m] += data[start[:m] + k]
    out = np.zeros(n)
    out[order] = acc
    return out


def entry_rows(M):
    return np.repeat(np.arange(M.shape[0]), np.diff(M.indptr))


def call(gsp, name, dtype, *args):
    import torch
    gsp._native.call(name + "_" + gsp._native.suffix(dtype), *args,
                     gsp._native.stream_ptr(torch.device("cuda")))


# ------------------------------------------------------------------ COO -> CSR assembly
RUN_LENGTHS = [1, 2, 3, 127, 128, 129, 1023, 1024, 1025]
KEYS_PER_LENGTH = 12
LONG_RUN = 200_000


def emission_case(dtype, seed=0):
    """Triplets whose keys repeat in runs of RUN_LENGTHS (KEYS_PER_LENGTH keys each) and one key
    LONG_RUN times, emitted interleaved in a random order, with values of mixed magnitude and
    sign so that the order of the sum shows in the last bits."""
    rng = np.random.default_rng(seed)
    n = 5000
    lengths = np.append(np.repeat(RUN_LENGTHS, KEYS_PER_LENGTH), LONG_RUN)
    keys = rng.choice(n * n - 2, lengths.size - 2, replace=False) + 1
    keys = np.append(keys, [0, n * n - 1])                 # (0, 0) and (n-1, n-1) too
    key = np.repeat(keys, lengths)
    spread = 4 if dtype == np.float32 else 10
    vals = (rng.standard_normal(key.size) * 10.0 ** rng.uniform(-spread, spread, key.size)).astype(dtype)
    emit = rng.permutation(key.size)
    key, vals = key[emit], vals[emit]
    return n, key // n, key % n, vals


def emission_order_sums(n, rows, cols, vals):
    """(indptr, indices, data) of the canonical CSR with each duplicate run summed sequentially
    in emission order in the value type: np.cumsum over the run, last value."""
    key = rows.astype(np.int64) * n + cols
    order = np.argsort(key, kind="stable")
    key, vals = key[order], vals[order]
    uniq, start = np.unique(key, return_index=True)
    end = np.append(start[1:], key.size)
    data = np.array([np.cumsum(vals[s:e], dtype=vals.dtype)[-1] for s, e in zip(start, end)],
                    dtype=vals.dtype)
    indptr = np.concatenate([[0], np.cumsum(np.bincount(uniq // n, minlength=n))])
    return indptr, uniq % n, data


@pytest.mark.parametrize("dtype", DTYPES)
def test_from_coo_sums_duplicates_in_emission_order(gsp, dtype):
    import torch
    n, rows, cols, vals = emission_case(dtype)
    indptr, indices, data = emission_order_sums(n, rows, cols, vals)
    structure = sparse.csr_matrix(sparse.coo_matrix((np.ones(len(rows)), (rows, cols)), shape=(n, n)))
    np.testing.assert_array_equal(indptr, structure.indptr)
    np.testing.assert_array_equal(indices, structure.indices)
    args = (torch.from_numpy(rows).cuda(), torch.from_numpy(cols).cuda(),
            torch.from_numpy(vals).cuda(), (n, n))
    D = gsp.graphs.DeviceCSR.from_coo(*args)
    np.testing.assert_array_equal(D.indptr.cpu().numpy(), indptr)
    np.testing.assert_array_equal(D.indices.cpu().numpy(), indices)
    got = D.data.cpu().numpy()
    run_len = np.bincount(np.unique(rows.astype(np.int64) * n + cols, return_inverse=True)[1])
    bad = bits(got) != bits(data)
    assert not bad.any(), "run lengths whose sum differs from the emission-order sum: {}".format(
        sorted(set(run_len[bad].tolist())))
    again = gsp.graphs.DeviceCSR.from_coo(*args)
    np.testing.assert_array_equal(bits(again.data.cpu().numpy()), bits(got))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("case", CASES)
def test_from_coo_moves_distinct_triplets(gsp, case, dtype):
    """Shuffled distinct triplets (stored zeros and -0.0 among them) land where SciPy puts them,
    values moved bit for bit."""
    import torch
    M = host(zoo(case), dtype)
    perm = np.random.default_rng(1).permutation(M.nnz)
    rows, cols, vals = entry_rows(M)[perm], M.indices[perm].astype(np.int64), M.data[perm]
    D = gsp.graphs.DeviceCSR.from_coo(torch.from_numpy(rows).cuda(), torch.from_numpy(cols).cuda(),
                                      torch.from_numpy(vals).cuda(), M.shape)
    assert_csr_bits(D, M, dtype)


OUT_OF_RANGE = [-1, 5, 2 ** 31, 2 ** 32 + 1, -2 ** 32 + 1, 2 ** 33]


@pytest.mark.parametrize("bad", OUT_OF_RANGE)
@pytest.mark.parametrize("where", ["rows", "cols"])
def test_from_coo_refuses_out_of_range_indices(gsp, where, bad):
    """Negative ids, ids >= n, and int64 ids that an int32 cast would wrap into [0, n)."""
    import torch
    n = 5
    rows = torch.tensor([0, 1, 2, 3, 4], device="cuda")
    cols = torch.tensor([1, 2, 3, 4, 0], device="cuda")
    (rows if where == "rows" else cols)[2] = bad
    vals = torch.ones(5, dtype=torch.float64, device="cuda")
    with pytest.raises(gsp._native.NativeError, match="out of range"):
        gsp.graphs.DeviceCSR.from_coo(rows, cols, vals, (n, n))
    with pytest.raises(gsp._native.NativeError, match="out of range"):
        gsp.graphs.Graph.from_coo(rows, cols, vals, n)
    if -2 ** 31 <= bad < 2 ** 31:                         # int32 ids take the same check
        with pytest.raises(gsp._native.NativeError, match="out of range"):
            gsp.graphs.DeviceCSR.from_coo(rows.int(), cols.int(), vals, (n, n))


@pytest.mark.parametrize("bad", [-1, 3, 2 ** 32 + 1, -2 ** 32 + 2])
def test_graph_refuses_out_of_range_int64_columns(gsp, bad):
    """A device (indptr, indices, data) triple with int64 columns: a column outside [0, n) is
    refused, also when an int32 cast would wrap it onto a valid, sorted column."""
    import torch
    indptr = torch.tensor([0, 1, 2, 3], dtype=torch.int32, device="cuda")
    indices = torch.tensor([1, bad, 1], dtype=torch.int64, device="cuda")
    data = torch.ones(3, dtype=torch.float64, device="cuda")
    with pytest.raises(ValueError, match="in range"):
        gsp.graphs.Graph((indptr, indices, data), dtype=np.float64)
    indices[1] = 2                                       # the same triple, in range, is accepted
    G = gsp.graphs.Graph((indptr.long(), indices, data), dtype=np.float64)
    np.testing.assert_array_equal(G.W.indices.cpu().numpy(), [1, 2, 1])


# ------------------------------------------------------------------ reshaping
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("case", CASES)
def test_transpose(gsp, case, dtype):
    M = host(zoo(case), dtype)
    T = M.T.tocsr()
    T.sort_indices()
    assert_csr_bits(device(gsp, M, dtype).transpose(), T, dtype)


def ref_symmetrize(M, method, dtype):
    """utils.symmetrize of M in dtype: the reference's formulas, sums in dtype; 'average' and
    'fill' halve that sum (SciPy halves it in float64, exactly, and the rounding to dtype is then
    the one of a halving in dtype); exact zeros dropped."""
    S = nno.symmetrize(M.astype(dtype), method).tocsr().astype(dtype)
    S.eliminate_zeros()
    S.sort_indices()
    return S


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("case", CASES)
def test_symmetrize(gsp, case, dtype, method):
    M = host(zoo(case), dtype)
    D = device(gsp, M, dtype)
    assert_csr_bits(D.symmetrize(method), ref_symmetrize(M, method, dtype), dtype)
    if method == "average":
        np.testing.assert_array_equal(orc.symmetrize_average(M).indices,
                                      ref_symmetrize(M, method, dtype).indices)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("case", CASES + ["nan"])
def test_eliminate_zeros(gsp, case, dtype):
    """Stored 0.0 and -0.0 go, NaN stays."""
    if case == "nan":
        M = _csr(4, [0, 0, 1, 2, 3, 3], [1, 3, 1, 2, 0, 3], [np.nan, 0.0, -0.0, np.nan, 1.0, -0.0])
    else:
        M = zoo(case)
    M = host(M, dtype)
    ref = M.copy()
    ref.eliminate_zeros()
    assert_csr_bits(device(gsp, M, dtype).eliminate_zeros(), ref, dtype)


# ------------------------------------------------------------------ induced submatrices
INDUCED_CASES = ["n1_loop", "path", "star", "directed", "isolated", "loop_only", "n1048579"]
INDUCED_KINDS = ["increasing", "unsorted", "repeated", "all", "one", "labels"]


def induced_ids(M, kind, rng):
    """(v, labels or None, increasing) of one induced-submatrix request on M."""
    n = M.shape[0]
    if kind == "all":
        return np.arange(n), None, True
    if kind == "one":
        diag = np.flatnonzero(M.diagonal())
        return np.array([diag[-1] if diag.size else n - 1]), None, True
    if kind == "labels":
        labels = rng.integers(0, 3, n)
        return np.lexsort((np.arange(n), labels)), labels, True
    m = max(1, n // 2)
    if kind == "increasing":
        return np.sort(rng.choice(n, m, replace=False)), None, True
    if kind == "unsorted":
        v = rng.choice(n, m, replace=False)
        if n > 1 and np.all(np.diff(v) > 0):
            v = v[::-1].copy()
        return v, None, False
    v = np.concatenate([rng.integers(0, n, m), [n - 1, n - 1, 0]])       # repeated
    return v, None, False


@pytest.mark.parametrize("kind", INDUCED_KINDS)
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("case", INDUCED_CASES)
def test_induced(gsp, case, dtype, kind):
    import torch
    from pygsp_b200.graphs.csr import row_ids
    M = host(zoo(case), dtype)
    v, labels, increasing = induced_ids(M, kind, np.random.default_rng(3))
    src = M
    if labels is not None:                     # entries whose two ends carry the same label
        r = entry_rows(M)
        keep = labels[r] == labels[M.indices]
        src = sparse.csr_matrix((M.data[keep], (r[keep], M.indices[keep])), shape=M.shape)
    ref = src[v][:, v].tocsr()
    ref.sort_indices()
    D = device(gsp, M, dtype)
    v_dev = torch.from_numpy(v.astype(np.int32)).cuda()
    lab_dev = None if labels is None else torch.from_numpy(labels.astype(np.int32)).cuda()
    S, rows = D.induced(v_dev, lab_dev, increasing)
    if increasing:
        assert rows is None
        assert_csr_bits(S, ref, dtype)
        return
    np.testing.assert_array_equal(rows.cpu().numpy(), row_ids(S.indptr).cpu().numpy())
    np.testing.assert_array_equal(S.indptr.cpu().numpy(), ref.indptr)
    C = gsp.graphs.DeviceCSR.from_coo(rows, S.indices, S.data, S.shape)
    assert_csr_bits(C, ref, dtype)


# ------------------------------------------------------------------ inspection
def ref_inspect(n, indptr, indices, data):
    """The seven counters of gsp_csr_inspect_*: NaN, Inf, negative, non-zero loop, stored zero,
    order violation (a column not above the previous one of its row), column out of range."""
    rows = np.repeat(np.arange(n), np.diff(indptr))
    prev = np.empty(len(indices), np.int64)
    prev[1:] = indices[:-1]
    starts = indptr[:-1][np.diff(indptr) > 0]
    prev[starts] = -1
    with np.errstate(invalid="ignore"):
        return [int(np.isnan(data).sum()), int(np.isinf(data).sum()), int((data < 0).sum()),
                int(((indices == rows) & (data != 0)).sum()), int((data == 0).sum()),
                int((indices <= prev).sum()), int(((indices < 0) | (indices >= n)).sum()), 0]


def run_inspect(gsp, n, indptr, indices, data, dtype):
    import torch
    stats = torch.full((8,), -7, dtype=torch.int64, device="cuda")
    call(gsp, "gsp_csr_inspect", dtype, gsp._native.i64(n),
         torch.from_numpy(np.asarray(indptr, np.int32)).cuda(),
         torch.from_numpy(np.asarray(indices, np.int32)).cuda(),
         torch.from_numpy(np.asarray(data, dtype)).cuda(), stats)
    return stats.cpu().numpy().tolist()


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("case", CASES)
def test_inspect_zoo(gsp, case, dtype):
    M = host(zoo(case), dtype)
    assert run_inspect(gsp, M.shape[0], M.indptr, M.indices, M.data, dtype) == \
        ref_inspect(M.shape[0], M.indptr, M.indices, M.data)


@pytest.mark.parametrize("dtype", DTYPES)
def test_inspect_counts_every_defect(gsp, dtype):
    """Each defect class, alone and together, on a well-formed indptr: NaN (also on the
    diagonal), +-Inf, negatives, stored 0.0 / -0.0, unsorted and repeated columns, and columns
    below 0 or at / past n (the int32 extremes included); an empty first and last row."""
    n = 7
    big = np.iinfo(np.int32)
    rows = [[], [1, 0, 3, 3], [2, -1, 7, int(big.max)], [int(big.min), 0, 6], [3, 2],
            [5, 4, 6], []]
    vals = [[], [np.nan, np.inf, -2.0, -0.0], [np.nan, 1.0, 0.0, -np.inf], [1.0, -0.0, 2.5],
            [0.0, 3.0], [2.0, -1.0, np.nan], []]
    indptr = np.concatenate([[0], np.cumsum([len(r) for r in rows])])
    indices = np.array(sum(rows, []), np.int64)
    data = np.array(sum(vals, []), np.float64).astype(dtype)
    want = ref_inspect(n, indptr, indices, data)
    assert want[:7] == [3, 2, 3, 3, 4, 6, 4]
    assert run_inspect(gsp, n, indptr, indices, data, dtype) == want


# ------------------------------------------------------------------ directedness, degrees
def ref_asymmetry(M):
    """Stored entries whose mirror is not stored or holds a different value."""
    n = M.shape[0]
    r, c = entry_rows(M).astype(np.int64), M.indices.astype(np.int64)
    key = r * n + c
    pos = np.searchsorted(key, c * n + r)
    found = pos < len(key)
    found[found] = key[pos[found]] == (c * n + r)[found]
    same = np.zeros(len(key), bool)
    same[found] = M.data[pos[found]] == M.data[found]
    return int((~same).sum())


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("case", CASES)
def test_asymmetry_count(gsp, case, dtype):
    import torch
    M = host(zoo(case), dtype)
    D = device(gsp, M, dtype)
    count = torch.full((1,), -7, dtype=torch.int64, device="cuda")
    call(gsp, "gsp_csr_asymmetry", dtype, gsp._native.i64(M.shape[0]), D.indptr, D.indices,
         D.data, count)
    assert int(count.item()) == ref_asymmetry(M)


def graph(gsp, case, dtype, lap_type="combinatorial"):
    return gsp.graphs.Graph(device(gsp, host(zoo(case), dtype), dtype), lap_type, dtype=dtype)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("case", CASES)
def test_graph_directedness_edges_and_degrees(gsp, case, dtype):
    """is_directed, n_edges and the degrees; dw bit-equal to the reference's sums, which add in
    stored order (column sums of W; the out-degree of a directed W summed in the same order)."""
    G = graph(gsp, case, dtype)
    W = canonical64(zoo(case), dtype)
    directed = orc.is_directed(W)
    assert G.is_directed() == directed
    assert G.n_edges == orc.count_edges(W, directed)
    assert G.W.nnz == W.nnz
    dw = orc.weighted_degree(W, directed)
    if directed:      # SciPy's row sums are pairwise: restate them in stored order
        np.testing.assert_allclose(G.dw, dw, rtol=1e-15, atol=0)
        dw = (np.asarray(W.sum(axis=0)).ravel() + seq_row_sums(W)) / 2
    else:
        np.testing.assert_array_equal(bits(seq_row_sums(W)), bits(dw))
    np.testing.assert_array_equal(bits(G.dw), bits(dw))
    np.testing.assert_array_equal(G.d, orc.degree(W, directed))


# ------------------------------------------------------------------ Laplacians
@pytest.mark.parametrize("lap_type", ["combinatorial", "normalized"])
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("case", CASES)
def test_laplacian(gsp, case, dtype, lap_type):
    G = graph(gsp, case, dtype, lap_type)
    W = canonical64(zoo(case), dtype)
    ref = orc.laplacian(W, lap_type)
    with np.errstate(invalid="ignore"):
        keep = ref.data.astype(dtype) != 0                # entries that round to 0 in dtype go
    r = entry_rows(ref)
    ref = sparse.csr_matrix((ref.data[keep], (r[keep], ref.indices[keep])), shape=ref.shape)
    L = G.L
    if lap_type == "combinatorial":
        np.testing.assert_array_equal(L.indptr.cpu().numpy(), ref.indptr)
        np.testing.assert_array_equal(L.indices.cpu().numpy(), ref.indices)
        got, want = L.data.cpu().numpy(), ref.data.astype(dtype)
        if dtype == np.float64:
            np.testing.assert_array_equal(bits(got), bits(want))
        else:
            assert np.all(np.abs(got.astype(np.float64) - want) <= np.spacing(np.abs(want)))
        return
    # normalized: CUDA pow is not libm pow.  Off the diagonal an entry is the product
    # -(d_i w_ij) d_j: same structure, and its own size is the scale.  The diagonal entry of a
    # loop is 1 - (d_i w_ii) d_i, whose terms are of size 1 + |L_ii|; it may cancel to a few ulp
    # of 1 on one side and to exactly 0 (not stored) on the other, so the diagonals are compared
    # as dense vectors.
    Lh = L.to_scipy().astype(np.float64)
    off_got, off_ref = sparse.triu(Lh, 1) + sparse.tril(Lh, -1), sparse.triu(ref, 1) + sparse.tril(ref, -1)
    off_got, off_ref = off_got.tocsr(), off_ref.tocsr()
    for a in (off_got, off_ref):
        a.sort_indices()
    np.testing.assert_array_equal(off_got.indptr, off_ref.indptr)
    np.testing.assert_array_equal(off_got.indices, off_ref.indices)
    n = ref.shape[0]
    d_got, d_ref = Lh.diagonal() if n else np.zeros(0), ref.diagonal() if n else np.zeros(0)
    got = np.concatenate([off_got.data, d_got])
    exact = np.concatenate([off_ref.data, d_ref])
    scale = np.concatenate([np.abs(off_ref.data), 1.0 + np.abs(d_ref)])
    nan = np.isnan(exact)
    np.testing.assert_array_equal(np.isnan(got), nan)
    got, exact, scale = got[~nan], exact[~nan], scale[~nan]
    tol = 8 * np.spacing(scale)
    if dtype == np.float32:               # and one float32 rounding of the result
        want = exact.astype(np.float32)
        tol = tol + np.spacing(np.abs(want)).astype(np.float64) + np.abs(want - exact)
    err = np.abs(got - exact)
    assert np.all(err <= tol), (err - tol).max()


# ------------------------------------------------------------------ spectral bounds
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("case", [c for c in CASES if c != "n0"])
def test_spectral_bounds(gsp, case, dtype):
    """The five raw outputs of gsp_spectral_bounds_* against graph.py:939-958 in NumPy on the
    same W, Ws and dw, then G._get_upper_bound() against the oracle's."""
    import torch
    G = graph(gsp, case, dtype)
    W, Ws, dw_dev = G.W, G._symmetric_adjacency(), G._degrees()[0]
    out = torch.empty(5, dtype=torch.float64, device="cuda")
    call(gsp, "gsp_spectral_bounds", dtype, gsp._native.i64(G.N), W.indptr, W.indices, W.data,
         Ws.indptr, Ws.indices, Ws.data, dw_dev, out)
    max_w, max_dw, max_edge, merris, n_nan = out.cpu().numpy()
    Wh, Wsh = W.to_scipy().astype(np.float64), Ws.to_scipy().astype(np.float64)
    dw = dw_dev.cpu().numpy()
    ninf = -np.inf
    assert max_w == (Wh.data.max() if Wh.nnz else ninf)
    assert max_dw == dw.max()
    assert max_edge == (np.max(dw[entry_rows(Wh)] + dw[Wh.indices]) if Wh.nnz else ninf)
    with np.errstate(divide="ignore", invalid="ignore"):
        t = dw + Wsh.dot(dw) / dw
        # the device product may contract to FMA: each row sum is within len * eps of its terms
        slack = (np.diff(Wsh.indptr) + 1) * np.finfo(np.float64).eps * \
            (abs(Wsh).dot(np.abs(dw)) / np.abs(dw))
    nan = np.isnan(t)
    assert n_nan == nan.sum()
    if nan.all():
        assert merris == ninf
    elif not np.isfinite(np.max(t[~nan])):
        assert merris == np.max(t[~nan])
    else:
        top = np.max(t[~nan])
        assert abs(merris - top) <= np.max(np.where(nan, 0, slack)) + 1e-15 * abs(top), (merris, top)
    W64 = canonical64(zoo(case), dtype)
    bound = G._get_upper_bound()
    rtol = 1e-14 if dtype == np.float64 or not G.is_directed() else 1e-6
    np.testing.assert_allclose(bound, orc.upper_bound(W64), rtol=rtol, atol=0)


# ------------------------------------------------------------------ row gather / scatter
@pytest.mark.parametrize("offset", [0, 1])
@pytest.mark.parametrize("width", [1, 2, 3, 4, 5, 8, 64, 67])
@pytest.mark.parametrize("dtype", DTYPES)
def test_gather_scatter_rows(gsp, dtype, width, offset):
    """dst = src[idx] and dst[idx] = src.  Row widths that are 16-byte multiples take the int4
    path when both bases are aligned; ``offset`` = 1 shifts both bases by one element, which
    forces the element-wise path."""
    import torch
    nat = gsp._native
    td = tdtype(dtype)
    rng = np.random.default_rng(width)
    n_src, n_idx = 1000, 777
    buf = torch.randn(offset + n_src * width, dtype=td, device="cuda")
    src = buf[offset:].view(n_src, width)
    idx = torch.from_numpy(rng.integers(0, n_src, n_idx)).cuda()     # repeats allowed
    idx[:2] = torch.tensor([0, n_src - 1])
    out = torch.full((offset + n_idx * width,), float("nan"), dtype=td, device="cuda")
    dst = out[offset:].view(n_idx, width)
    call(gsp, "gsp_gather_rows", dtype, nat.i64(n_idx), idx, src, nat.i64(width), dst)
    assert torch.equal(dst, src[idx])
    assert torch.isnan(out[:offset]).all()

    perm = torch.from_numpy(rng.permutation(n_src)[:n_idx]).cuda()   # distinct targets
    vals = torch.randn(offset + n_idx * width, dtype=td, device="cuda")[offset:].view(n_idx, width)
    out = torch.full((offset + n_src * width,), float("nan"), dtype=td, device="cuda")
    dst = out[offset:].view(n_src, width)
    call(gsp, "gsp_scatter_rows", dtype, nat.i64(n_idx), perm, vals, nat.i64(width), dst)
    want = torch.full_like(dst, float("nan"))
    want[perm] = vals
    assert torch.equal(torch.nan_to_num(dst, 7.0), torch.nan_to_num(want, 7.0))
    assert torch.isnan(out[:offset]).all()


# ------------------------------------------------------------------ products on heavy / empty rows
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("case", ["n1", "n1_loop", "n1000_nnz0", "star", "isolated", "loop_only",
                                  "n1048579"])
def test_dot_heavy_and_empty_rows(gsp, case, dtype):
    """SpMV and SpMM on a 70 000-entry row and on empty rows.  With small integers as weights and
    signal every partial sum is an integer below 2^24, so any summation order is exact and the
    products must equal SciPy's bit for bit: a term lost or counted twice shows.  The zoo's own
    weights then meet the SpMV tolerance of the other SpMV tests."""
    M = host(zoo(case), dtype)
    rng = np.random.default_rng(4)
    Mi = M.copy()
    Mi.data = (np.arange(M.nnz) % 7 - 3).astype(dtype)
    Di = device(gsp, Mi, dtype)
    for x in (rng.integers(-4, 5, M.shape[1]), rng.integers(-4, 5, (M.shape[1], 5))):
        x = x.astype(dtype)
        got, ref = Di.dot(x), Mi.astype(np.float64).dot(x.astype(np.float64))
        assert got.shape == ref.shape
        np.testing.assert_array_equal(got, ref)
    x = rng.standard_normal(M.shape[1])
    got, ref = device(gsp, M, dtype).dot(x), M.astype(np.float64).dot(x)
    scale = max(np.abs(ref).max(), 1e-30)
    assert np.abs(got - ref).max() / scale <= (2e-6 if dtype == np.float32 else 1e-13)
