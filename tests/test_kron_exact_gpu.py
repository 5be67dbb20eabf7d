"""The exact Kron reduction and the sparsifier's kernels at their edges (csrc/schur.cu,
pygsp_b200/reduction.py _split, _removed_components, _schur, graph_sparsify), against host
restatements (oracle/kron_exact_oracle.py): the component structure against SciPy, the one-CTA
Schur kernel called directly at every thread-loop and shared-memory boundary, the dense fallback's
gather, the whole reduction with small, dense and neighbour-less components mixed, and every
sampler count replayed from Philox.  Exactly representable cases are compared bit for bit, the
others within the bound of keo.C_BOUND."""
import time
import types

import numpy as np
import pytest
from scipy import sparse

from oracle import kron_exact_oracle as keo
from oracle import multiresolution_oracle as mro

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gsp():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import pygsp_b200
    return pygsp_b200


def _smem(s, b):
    """Dynamic shared memory of one component, as _schur computes it."""
    return 8 * (s * s + s + s * b) + 4 * b


def _device(gsp, M, ind):
    """_split and _removed_components of (M, ind) on the device, as _schur calls them; ``slot0``
    is slot as _split left it."""
    red = gsp.reduction
    _, dev = red._ctx()
    Md = red._device_matrix(M, dev)
    ind = np.asarray(ind, dtype=np.int64)
    slot, rem, R, r_rows = red._split(Md, ind)
    slot0 = slot.clone()
    nc, cvert, cptr, sizes, comp_of, bidx, nbs, bptr = red._removed_components(Md, slot, rem,
                                                                               ind.size)
    return types.SimpleNamespace(M=Md, ind=ind, slot0=slot0, slot=slot, rem=rem, R=R,
                                 r_rows=r_rows, nc=nc, cvert=cvert, cptr=cptr, sizes=sizes,
                                 comp_of=comp_of, bidx=bidx, nbs=nbs, bptr=bptr)


def _host(t):
    return t.cpu().numpy()


# ------------------------------------------------------------------ component structure ----
def _check_structure(gsp, M, ind):
    M = sparse.csr_matrix(M)
    n, m = M.shape[0], len(ind)
    D = _device(gsp, M, ind)
    kept_index = np.full(n, -1, dtype=np.int64)
    kept_index[ind] = np.arange(m)
    kept = kept_index >= 0
    np.testing.assert_array_equal(_host(D.slot0), np.where(kept, -1 - kept_index, 0))
    np.testing.assert_array_equal(_host(D.rem), np.flatnonzero(~kept))
    R = sparse.csr_matrix((_host(D.R.data), (_host(D.r_rows), _host(D.R.indices))), shape=(m, m))
    want_R = M[ind][:, ind]
    assert R.nnz == want_R.nnz and (R != want_R).nnz == 0

    # components in increasing order of their smallest vertex (gsp_component_order sorts by the
    # union-find root, the smallest vertex): the mixed reduction below relies on that order
    comps = keo.removed_components(M, ind)
    assert D.nc == len(comps)
    cvert, cptr, sizes = _host(D.cvert), _host(D.cptr), _host(D.sizes)
    bidx, bptr, nbs = _host(D.bidx), _host(D.bptr), _host(D.nbs)
    slot, comp_of = _host(D.slot), _host(D.comp_of)
    assert cptr[0] == 0 and cptr[-1] == n - m and bptr[0] == 0 and bptr[-1] == bidx.size
    want_of = np.full(n, -1, dtype=np.int64)
    for c, comp in enumerate(comps):
        v = cvert[cptr[c]:cptr[c + 1]]
        np.testing.assert_array_equal(np.sort(v), comp["vertices"])
        assert sizes[c] == v.size
        np.testing.assert_array_equal(slot[v], np.arange(v.size))
        np.testing.assert_array_equal(bidx[bptr[c]:bptr[c + 1]], comp["kept"])
        assert nbs[c] == comp["kept"].size
        want_of[v] = c
    np.testing.assert_array_equal(comp_of, want_of)
    np.testing.assert_array_equal(comp_of == -1, kept)
    np.testing.assert_array_equal(slot[ind], -1 - np.arange(m))
    return comps


@pytest.mark.parametrize("seed", [0, 1])
def test_component_structure_of_built_graphs(gsp, seed):
    specs = [(1, 1, "well"), (3, 0, "well"), (17, 9, "ill"), (2, 1, "well"), (64, 126, "well"),
             (5, 4, "indefinite"), (65, 10, "well"), (1, 2, "well"), (8, 300, "ill")]
    M, ind, built = keo.build_components(specs, seed=seed)
    comps = _check_structure(gsp, M, ind)
    for got, want in zip(comps, built):
        np.testing.assert_array_equal(got["vertices"], want["vertices"])
        np.testing.assert_array_equal(got["kept"], want["kept"])


def test_component_structure_of_a_sensor_graph(gsp):
    G = gsp.graphs.Sensor(20_000, k=10, seed=3, dtype=np.float64, order="morton")
    L = G.L.to_scipy().astype(np.float64).tocsr()
    ind = np.random.default_rng(5).permutation(G.N)[:12_000]      # keep 60 %, in random order
    comps = _check_structure(gsp, L, ind)
    sizes = np.array([c["vertices"].size for c in comps])
    print("%d components, largest %d, %d without kept neighbours"
          % (len(comps), sizes.max(), sum(c["kept"].size == 0 for c in comps)))
    assert len(comps) >= 50 and sizes.max() > gsp.reduction.SMALL_MAX


# ------------------------------------------------------------------ gsp_schur_small_f64 ----
def _schur_small(gsp, D, comps):
    """gsp_schur_small_f64 on the components ``comps`` of D, with the shared memory _schur would
    pass: (rows, cols, vals, status, out_off) on the host.  Slots of the other components keep
    -7 / NaN."""
    import torch
    from pygsp_b200 import _native as nat
    dev = D.M.device
    sizes, nbs = _host(D.sizes), _host(D.nbs)
    comps = np.asarray(comps, dtype=np.int32)
    smem = max(_smem(int(sizes[c]), int(nbs[c])) for c in comps)
    off = np.zeros(D.nc + 1, dtype=np.int64)
    off[1:] = np.cumsum(nbs * nbs)
    total = int(off[-1])
    rows = torch.full((total,), -7, dtype=torch.int32, device=dev)
    cols = torch.full((total,), -7, dtype=torch.int32, device=dev)
    vals = torch.full((total,), float("nan"), dtype=torch.float64, device=dev)
    status = torch.full((1,), 5, dtype=torch.int32, device=dev)
    nat.call("gsp_schur_small_f64", D.M.indptr, D.M.indices, D.M.data, D.slot, D.cvert, D.cptr,
             D.bptr.to(torch.int32), D.bidx, nat.i64(comps.size),
             torch.from_numpy(comps).to(dev), nat.i32(smem), torch.from_numpy(off).to(dev),
             rows, cols, vals, status, nat.stream_ptr())
    return _host(rows), _host(cols), _host(vals), int(status.item()), off


def _block(out, c):
    rows, cols, vals, _, off = out
    o0, o1 = off[c], off[c + 1]
    b = int(round(np.sqrt(o1 - o0)))
    return rows[o0:o1], cols[o0:o1], vals[o0:o1].reshape(b, b)


def _check_blocks(out, blocks, kinds=None, which=None):
    """The triplets of every component (or of those in ``which``): rows / cols bit for bit,
    row-major over B in kept-index order; the values exactly symmetric and within keo.block_bound
    of the host block ('well' components also within 1e-13 of their largest entry).  Returns the
    largest error / bound."""
    worst = 0.0
    for c in range(len(blocks)) if which is None else which:
        blk = blocks[c]
        r, cc, V = _block(out, c)
        k = blk["kept"]
        np.testing.assert_array_equal(r, np.repeat(k, k.size))
        np.testing.assert_array_equal(cc, np.tile(k, k.size))
        np.testing.assert_array_equal(V, V.T)
        if k.size == 0:
            continue
        want = blk["block"]
        err = float(np.abs(V - want).max())
        bound = keo.block_bound(blk)
        assert err <= bound, (c, blk["vertices"].size, k.size, err, bound)
        if kinds is not None and kinds[c] == "well":
            assert err <= 1e-13 * np.abs(want).max(), (c, err)
        worst = max(worst, err / bound)
    return worst


SMALL_CASES = {
    # (s, b): s = 1 and 2 edges, the trailing update crossing 256 entries in the first column
    # (m^2 = 256 at s = 17, 289 at s = 18), the 96 KiB budget at s = 64, b = 126 (98 296 bytes,
    # above 48 KiB), the solve loop wrapping and 90 000 outputs at b = 300, and 188 080 bytes at
    # s = 64, b = 300, which only a direct call reaches
    "s1": [(1, 1, "well"), (1, 2, "well"), (1, 1, "well"), (1, 2, "well")],
    "s2": [(2, 1, "well"), (2, 1, "ill"), (2, 3, "well")],
    "s17_s18": [(17, 9, "well"), (17, 9, "ill"), (18, 9, "well"), (18, 40, "ill")],
    "s64_b126": [(64, 126, "well"), (3, 2, "well"), (64, 126, "ill")],
    "s8_b300": [(8, 300, "well"), (8, 300, "ill")],
    "s64_b300": [(64, 300, "well"), (5, 7, "ill"), (64, 300, "ill")],
}


@pytest.mark.parametrize("name", sorted(SMALL_CASES))
def test_schur_small_blocks(gsp, name):
    specs = SMALL_CASES[name]
    M, ind, _ = keo.build_components(specs, seed=11)
    D = _device(gsp, M, ind)
    blocks = keo.schur_blocks(M, ind)
    out = _schur_small(gsp, D, np.arange(D.nc))
    assert out[3] == 0
    worst = _check_blocks(out, blocks, [k for _, _, k in specs])
    print("%s: smem %d bytes, largest error / bound %.2e"
          % (name, max(_smem(s, b) for s, b, _ in specs), worst))


def test_schur_small_exact_blocks_on_many_ctas(gsp):
    """A path of 200 001 vertices with weight-2 edges and every odd vertex removed: 10^5
    components with s = 1, diagonal 4 and two kept neighbours, so C = 2, Y = -1 and every block is
    exactly -[[1, 1], [1, 1]].  Then 60 hubs (s = 1) with diagonals 4^k and integer weights to 1 to
    40 kept vertices of the path: Y = -w / 2^k and every entry -w_i w_j / 4^k is exact."""
    n = 200_001
    rng = np.random.default_rng(2)
    v = np.arange(n - 1)
    rows, cols, vals = list(v), list(v + 1), [2.0] * (n - 1)
    diag = [4.0] * n
    hub_b = np.r_[np.arange(1, 41), rng.integers(1, 41, 20)]
    for h, b in enumerate(hub_b):
        nb = 2 * rng.choice(n // 2 + 1, b, replace=False)
        rows += [n + h] * b
        cols += list(nb)
        vals += list(rng.integers(1, 8, b).astype(np.float64))
        diag.append(4.0 ** rng.integers(1, 7))
    N = n + hub_b.size
    W = sparse.coo_matrix((vals, (rows, cols)), shape=(N, N)).tocsr()
    M = (sparse.diags(np.array(diag)) - W - W.T).tocsr()
    ind = np.arange(0, n, 2)
    D = _device(gsp, M, ind)
    assert D.nc == n // 2 + hub_b.size
    out = _schur_small(gsp, D, np.arange(D.nc))
    rows_o, cols_o, vals_o, status, off = out
    assert status == 0
    npath = n // 2
    np.testing.assert_array_equal(off[:npath + 1], 4 * np.arange(npath + 1))
    k = np.arange(npath)
    np.testing.assert_array_equal(rows_o[:4 * npath].reshape(-1, 4),
                                  np.stack([k, k, k + 1, k + 1], 1))
    np.testing.assert_array_equal(cols_o[:4 * npath].reshape(-1, 4),
                                  np.stack([k, k + 1, k, k + 1], 1))
    assert np.all(vals_o[:4 * npath] == -1.0)
    for h in range(hub_b.size):
        c = npath + h
        hub = n + h
        nbr = M[hub].indices[M[hub].indices != hub]
        kept = np.sort(nbr // 2)
        m = np.asarray(M[hub, 2 * kept].toarray()).ravel()
        want = -np.outer(m, m) / M[hub, hub]
        r, cc, V = _block(out, c)
        np.testing.assert_array_equal(r, np.repeat(kept, kept.size))
        np.testing.assert_array_equal(cc, np.tile(kept, kept.size))
        np.testing.assert_array_equal(V, want)


def test_schur_small_status_leaves_other_blocks_alone(gsp):
    """One indefinite component among twenty good ones: status 1, every output finite, and the good
    components' triplets bit for bit those of a call without the bad one."""
    specs = ([(6, 5, "well"), (9, 7, "ill")] * 5 + [(5, 4, "indefinite")]
             + [(12, 20, "well"), (4, 3, "ill")] * 5)
    M, ind, _ = keo.build_components(specs, seed=6)
    D = _device(gsp, M, ind)
    bad = 10
    assert specs[bad][2] == "indefinite" and D.nc == 21
    full = _schur_small(gsp, D, np.arange(D.nc))
    assert full[3] == 1
    assert np.all(np.isfinite(full[2]))
    good = np.r_[np.arange(bad), np.arange(bad + 1, D.nc)]
    part = _schur_small(gsp, D, good)
    assert part[3] == 0
    for c in good:
        for a, b in zip(_block(full, c), _block(part, c)):
            np.testing.assert_array_equal(a, b)
    _, _, V = _block(part, bad)
    assert np.all(np.isnan(V))                          # the bad block was not run
    _check_blocks(part, keo.schur_blocks(M, ind), which=good)


# ------------------------------------------------------------------ dense fallback ---------
def test_schur_gather_copies_the_blocks(gsp):
    """gsp_schur_gather_f64 writes M[S][:, S] and M[S][:, B] bit for bit (S in the component's
    slot order), for s = 65, 129 and 300 (three 128-thread CTAs)."""
    import torch
    from pygsp_b200 import _native as nat
    specs = [(65, 10, "well"), (129, 40, "ill"), (300, 77, "well")]
    M, ind, _ = keo.build_components(specs, seed=8)
    D = _device(gsp, M, ind)
    cptr, bptr, cvert = (_host(t).astype(np.int64) for t in (D.cptr, D.bptr, D.cvert))
    for c, (s, b, _) in enumerate(specs):
        c0, c1, b0, b1 = int(cptr[c]), int(cptr[c + 1]), int(bptr[c]), int(bptr[c + 1])
        A = torch.full((s, s), float("nan"), dtype=torch.float64, device=D.M.device)
        B = torch.full((s, b), float("nan"), dtype=torch.float64, device=D.M.device)
        nat.call("gsp_schur_gather_f64", D.M.indptr, D.M.indices, D.M.data, D.slot,
                 D.cvert[c0:c1], nat.i64(s), D.bidx[b0:b1], nat.i64(b), A, B, nat.stream_ptr())
        S = cvert[c0:c1]
        Bv = ind[_host(D.bidx)[b0:b1]]
        np.testing.assert_array_equal(_host(A), M[S][:, S].toarray())
        np.testing.assert_array_equal(_host(B), M[S][:, Bv].toarray())


# in component order: small, dense (s = 65), dense (s = 64, b = 127: 98 812 bytes), no kept
# neighbour, small, ... twice, the second time ill-conditioned
MIXED = [(5, 6, "well"), (65, 10, "well"), (64, 127, "well"), (6, 0, "well"), (4, 3, "well"),
         (9, 20, "ill"), (65, 12, "ill"), (64, 127, "ill"), (7, 0, "well"), (2, 1, "ill"),
         (1, 2, "well")]


@pytest.fixture(scope="module")
def mixed():
    M, ind, comps = keo.build_components(MIXED, seed=9)
    blocks = keo.schur_blocks(M, ind)
    return M, ind, blocks, mro.kron_matrix(M, ind), keo.schur_tolerance(M, ind, blocks)


def test_mixed_small_and_dense_reduction(gsp, mixed, monkeypatch):
    red = gsp.reduction
    M, ind, blocks, want, tol = mixed
    paths = ["small" if s <= red.SMALL_MAX and _smem(s, b) <= red._SMALL_SMEM and b > 0
             else "dense" if b > 0 else "none" for s, b, _ in MIXED]
    assert paths == ["small", "dense", "dense", "none", "small", "small", "dense", "dense", "none",
                     "small", "small"]
    names = []
    call = red._call
    monkeypatch.setattr(red, "_call", lambda name, *a: (names.append(name), call(name, *a)))
    got = red.kron_reduction(M, ind).toarray()
    assert names.count("gsp_schur_small_f64") == 1 and names.count("gsp_schur_gather_f64") == 4
    err = np.abs(got - want)
    print("mixed: largest error / tolerance %.2e" % (err / np.where(tol > 0, tol, 1)).max())
    assert np.all(err <= tol)
    monkeypatch.setattr(red, "SMALL_MAX", 0)
    names.clear()
    dense = red.kron_reduction(M, ind).toarray()
    assert "gsp_schur_small_f64" not in names and names.count("gsp_schur_gather_f64") == 9
    assert np.all(np.abs(dense - want) <= tol)


def test_kept_order_permutes_the_result_exactly(gsp, mixed):
    """Components, their order, each entry's terms and the order in which duplicates are summed
    do not depend on the order of ind: kron_reduction(M, ind[p]) = P K P^T bit for bit."""
    M, ind, _, _, _ = mixed
    K = gsp.reduction.kron_reduction(M, ind).toarray()
    p = np.random.default_rng(4).permutation(ind.size)
    Kp = gsp.reduction.kron_reduction(M, ind[p]).toarray()
    np.testing.assert_array_equal(Kp, K[np.ix_(p, p)])


def test_float32_graph_is_the_float64_result_rounded(gsp):
    """Integer weights make the float32 and float64 Laplacians equal, so kron_reduction of the
    float32 graph is the float64 graph's reduced W rounded to float32, bit for bit."""
    P = gsp.graphs.Sensor(600, k=6, seed=3, dtype=np.float64).W.to_scipy()
    T = sparse.triu(P, 1).tocoo()
    w = np.random.default_rng(1).integers(1, 6, T.nnz).astype(np.float64)
    W = sparse.coo_matrix((w, (T.row, T.col)), shape=P.shape).tocsr()
    W = (W + W.T).tocsr()
    G64 = gsp.graphs.Graph(W, dtype=np.float64)
    G32 = gsp.graphs.Graph(W, dtype=np.float32)
    assert (G32.L.to_scipy().astype(np.float64) != G64.L.to_scipy()).nnz == 0
    ind = np.random.default_rng(2).permutation(W.shape[0])[:250]
    K32 = gsp.reduction.kron_reduction(G32, ind)
    K64 = gsp.reduction.kron_reduction(G64, ind)
    W32 = K32.W.to_scipy()
    assert W32.dtype == np.float32
    np.testing.assert_array_equal(W32.toarray(), K64.W.to_scipy().toarray().astype(np.float32))


@pytest.mark.parametrize("b,path", [(8190, "small"), (8191, "dense")])
def test_hub_at_the_shared_memory_budget(gsp, b, path, monkeypatch):
    """One removed hub (s = 1, diagonal 4^7) joined with integer weights 1..3 to b kept vertices of
    diagonal 8: the b^2 block -w w^T / 2^14 and its sum with the diagonal are exact.  b = 8190 needs
    98 296 bytes and is one CTA writing 67 M triplets; b = 8191 needs 98 308 and goes dense."""
    import torch
    free, _ = torch.cuda.mem_get_info()
    if free < 4 * 2 ** 30:
        pytest.skip("needs 4 GB of free device memory")
    red = gsp.reduction
    assert (_smem(1, b) <= red._SMALL_SMEM) == (path == "small")
    w = np.random.default_rng(b).integers(1, 4, b).astype(np.float64)
    k = np.arange(1, b + 1)
    M = sparse.csr_matrix((np.r_[16384.0, -w, -w, np.full(b, 8.0)],
                           (np.r_[0, np.zeros(b, int), k, k], np.r_[0, k, np.zeros(b, int), k])),
                          shape=(b + 1, b + 1))
    names = []
    call = red._call
    monkeypatch.setattr(red, "_call", lambda name, *a: (names.append(name), call(name, *a)))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    K = red._schur(red._device_matrix(M, torch.device("cuda")), k)
    torch.cuda.synchronize()
    print("hub b = %d (%s): %.2f s" % (b, path, time.perf_counter() - t0))
    assert ("gsp_schur_small_f64" in names) == (path == "small")
    assert ("gsp_schur_gather_f64" in names) == (path == "dense")
    np.testing.assert_array_equal(_host(K.indptr), np.arange(b + 1, dtype=np.int64) * b)
    np.testing.assert_array_equal(_host(K.indices).reshape(b, b),
                                  np.broadcast_to(np.arange(b), (b, b)))
    want = -np.outer(w, w) / 16384.0
    want[np.diag_indices(b)] += 8.0
    np.testing.assert_array_equal(_host(K.data).reshape(b, b), want)


# ------------------------------------------------------------------ the sampler -----------
def _sample(gsp, k, q, seed):
    import torch
    from pygsp_b200 import _native as nat
    k = np.asarray(k, dtype=np.uint64)
    kt = torch.from_numpy(k.view(np.int64)).cuda()
    counts = torch.full((k.size,), -1, dtype=torch.int64, device=kt.device)
    nat.call("gsp_sparsify_sample", nat.i64(k.size), kt, nat.i64(q), nat.u64(seed), counts,
             nat.stream_ptr())
    return _host(counts)


def _weights(name):
    rng = np.random.default_rng(3)
    if name == "random":
        return rng.integers(0, 1000, 5000)
    if name == "zeros":                       # zero at the first and last position and in runs
        k = rng.integers(1, 1000, 5000)
        k[0] = k[-1] = 0
        k[100:140] = 0
        k[2000:2001] = 0
        k[4990:4999] = 0
        return k
    if name == "one_edge":
        return np.array([12345])
    if name == "2^32_each":                   # T = 2^32 10^6, near 2^52: many scan tiles
        return np.full(10 ** 6, 2 ** 32, dtype=np.uint64)
    if name == "near_2^63":
        k = [int(v) for v in rng.integers(2 ** 50, 2 ** 51, 3000)]
        return np.array(k + [2 ** 63 - 1 - sum(k)], dtype=np.uint64)
    return np.array({"ones": [1, 1, 1], "gap": [1, 0, 2], "single3": [3]}[name])


SAMPLER_CASES = [("random", q) for q in (0, 1, 2, 127, 128, 129, 255, 16_385, 10 ** 6 + 3)] + [
    ("one_edge", 1000), ("zeros", 16_385), ("zeros", 10 ** 6 + 3), ("2^32_each", 10 ** 6 + 3),
    ("near_2^63", 16_385), ("ones", 16_385), ("gap", 16_385), ("single3", 1000)]


@pytest.mark.parametrize("name,q", SAMPLER_CASES)
def test_sampler_counts_are_the_replay(gsp, name, q):
    k = _weights(name)
    seed = 0x9E3779B97F4A7C15 ^ q
    got = _sample(gsp, k, q, seed)
    np.testing.assert_array_equal(got, keo.sparsify_counts(k, q, seed))
    assert got.sum() == q


def test_graph_sparsify_weights_are_the_replayed_counts(gsp, monkeypatch):
    """graph_sparsify on a 3000-vertex sensor graph, the (k, q, seed) handed to the sampler
    recorded: the device counts are the replay, and every returned weight is
    count w / (q P_e), P_e = k_e / sum k, in the same float64 operations, bit for bit.  (PyTorch
    divides a tensor by a Python number as a product with its reciprocal: P_e = k_e (1 / sum k).)"""
    red = gsp.reduction
    G = gsp.graphs.Sensor(3000, k=10, seed=6, dtype=np.float64, order="morton")
    calls = []
    call = red._call

    def record(name, *args):
        call(name, *args)
        if name == "gsp_sparsify_sample":
            calls.append((_host(args[1]).copy(), args[2].value, args[3].value,
                          _host(args[4]).copy()))
    monkeypatch.setattr(red, "_call", record)
    S = red.graph_sparsify(G, 0.3, seed=11)
    assert calls
    for k, q, seed, counts in calls:
        np.testing.assert_array_equal(counts, keo.sparsify_counts(k, q, seed))
    k, q, seed, counts = calls[-1]
    L = G.L.to_scipy().astype(np.float64).tocoo()
    edge = (L.row > L.col) & (-L.data >= 1e-10)
    s, e, w = L.row[edge], L.col[edge], -L.data[edge]
    order = np.lexsort((e, s))                       # graph_sparsify's CSR order
    s, e, w = s[order], e[order], w[order]
    assert k.size == s.size
    counts = keo.sparsify_counts(k, q, seed)
    Pe = k.astype(np.float64) * (1.0 / int(k.sum()))
    hit = counts > 0
    want = counts[hit].astype(np.float64) * w[hit] / (q * Pe[hit])
    Ws = S.W.to_scipy().astype(np.float64).tocsr()
    assert Ws.nnz == 2 * int(hit.sum())
    np.testing.assert_array_equal(np.asarray(Ws[s[hit], e[hit]]).ravel(), want)
    np.testing.assert_array_equal(np.asarray(Ws[e[hit], s[hit]]).ravel(), want)


# ------------------------------------------------------------------ gsp_edge_resistance_f64
@pytest.mark.parametrize("lda_pad", [0, 5])
def test_edge_resistance_bitwise(gsp, lda_pad):
    """R_e = (A[u,u] + A[v,v]) - (A[u,v] + A[v,u]) bit for bit on a random non-symmetric A, with
    lda = N and lda = N + 5, over edges that touch row and column N - 1.  Offsets past 2^31
    elements (a 16 GB matrix) are not tested."""
    import torch
    from pygsp_b200 import _native as nat
    n, lda = 700, 700 + lda_pad
    rng = np.random.default_rng(lda)
    A = rng.standard_normal((n, lda))
    u = rng.integers(0, n, 5000)
    v = rng.integers(0, n, 5000)
    u = np.r_[u, n - 1, 0, n - 1, n - 2, n - 1, 3]
    v = np.r_[v, 0, n - 1, n - 2, n - 1, n - 1, 3]
    dev = torch.device("cuda")
    R = torch.full((u.size,), float("nan"), dtype=torch.float64, device=dev)
    nat.call("gsp_edge_resistance_f64", nat.i64(u.size),
             torch.from_numpy(u.astype(np.int32)).to(dev),
             torch.from_numpy(v.astype(np.int32)).to(dev), torch.from_numpy(A).to(dev),
             nat.i64(lda), R, nat.stream_ptr())
    want = (A[u, u] + A[v, v]) - (A[u, v] + A[v, u])
    np.testing.assert_array_equal(_host(R), want)
