"""The tiled float32 Chebyshev step (csrc/cheby_tiled.cu), row by row.

Every element of a single step is checked against the float64 reference of
oracle/step_oracle.py, within its proven error bound, on graphs built so that each path of the
kernel runs: the last tile ending at nnz for every residue nnz % 4, tiles with empty CSR slabs,
graphs smaller than one tile, a hub that shrinks the ring, scattered gathers, weights over many
decades, and a graph large enough for every CTA to go around its shared-memory ring more than
twice.  Whole calls are checked against the oracle, and the outputs of every launch variant (lane
mapping, staging mode, ring depth, warps, CTAs per SM, L2 hint, sweep direction, shared-memory
budget, tile height, halo-capable instantiation) and of the row-group kernel must be the same
bits.
"""
import numpy as np
import pytest
from scipy import sparse

from conftest import relerr_cols
from oracle import pygsp_oracle as orc
from oracle import step_oracle as so

pytestmark = pytest.mark.gpu

F32_TOL = 1e-5
NSIGS = (8, 16, 32, 64, 128)
NSCALES = (0, 1, 2, 3, 16)
NAN32 = 0x7FE5A5A5                 # quiet NaN with a payload: rows a step must not touch
NAN64 = 0x7FFA5A5A5A5A5A5A


def _default_r(nsig, nscales):
    """Rows per tile that gsp_cheby_tile_plan picks without GSPB200_TILE_R."""
    R = 64 if nscales <= 1 else (32 if nscales <= 2 else 16)
    if nsig == 128:
        R = max(8, R // 2)
    if nsig <= 16:
        R = max(R, 16 * (128 // nsig))
    return R


@pytest.fixture(scope="module")
def gsp():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import pygsp_b200
    return pygsp_b200


# --------------------------------------------------------------------------- catalogue
def _force_nnz_mod4(W, t, rng):
    """Tweak W so that its Laplacian stores nnz = t (mod 4): isolating a vertex of degree d
    removes 2d + 1 entries, adding an edge adds 2."""
    W = sparse.lil_matrix(W)
    n = W.shape[0]
    for _ in range(3):
        L = orc.laplacian(sparse.csr_matrix(W))
        d = (L.nnz - t) % 4
        if d == 0:
            return sparse.csr_matrix(W)
        deg = np.diff(L.indptr) - 1
        if d == 2:
            while True:
                a, b = rng.integers(n // 3, 2 * n // 3, 2)
                if a != b and L[a, b] == 0:
                    W[a, b] = W[b, a] = 0.5
                    break
        else:
            want = 0 if d == 1 else 1
            v = next(int(v) for v in rng.permutation(np.arange(n // 3, 2 * n // 3))
                     if deg[v] > 0 and deg[v] % 2 == want)
            W[v, :] = 0
            W[:, v] = 0
    raise AssertionError("nnz residue not reached")


def _laplacian32(W, lap_type="combinatorial"):
    L = orc.laplacian(sparse.csr_matrix(W), lap_type).astype(np.float32)
    L.eliminate_zeros()
    L.sort_indices()
    return L


def _build_catalogue():
    rng = np.random.default_rng(2024)
    cat = {}
    base = so.sensor_adjacency(4096, k=8, seed=21)
    for t in range(4):
        cat["nnz%%4=%d" % t] = _laplacian32(_force_nnz_mod4(base, t, rng))
    # runs of 600 isolated vertices (>= 2R for every R a plan picks) at the start, middle, end
    W0 = _force_nnz_mod4(so.sensor_adjacency(3000, k=8, seed=22), 2, rng).tocoo()
    place = np.concatenate([np.arange(600, 2100), np.arange(2700, 4200)])
    cat["isolated runs"] = _laplacian32(sparse.coo_matrix(
        (W0.data, (place[W0.row], place[W0.col])), shape=(4800, 4800)))
    # a hub of 3000 neighbours beside rows of two to four entries
    n = 8192
    ends = [(np.arange(0, n, 2), np.arange(1, n, 2)), (np.arange(1, n - 2, 16), np.arange(2, n - 1, 16))]
    nbrs = rng.choice(np.setdiff1d(np.arange(n), [4099]), 3000, replace=False)
    ends.append((np.full(3000, 4099), nbrs))
    r = np.concatenate([e[0] for e in ends])
    c = np.concatenate([e[1] for e in ends])
    H = sparse.coo_matrix((rng.uniform(0.5, 1.5, r.size), (r, c)), shape=(n, n)).tocsr()
    cat["hub"] = _laplacian32(H + H.T)
    # the Sensor graph renumbered at random: scattered gathers
    p = rng.permutation(4096)
    cat["renumbered"] = _laplacian32(base[p][:, p])
    # weights over more than six decades; self-loops + normalized; directed
    T = sparse.triu(base, 1).tocsr()
    T.data = T.data * 10.0 ** rng.uniform(-6.5, 0, T.nnz)
    wide = (T + T.T).tocsr()
    cat["wide weights"] = _laplacian32(wide)
    loops = wide + sparse.diags(np.where(rng.uniform(size=4096) < 0.3, rng.uniform(0.1, 2, 4096), 0))
    cat["self-loops, normalized"] = _laplacian32(loops, "normalized")
    D = base.copy()
    D.data = D.data * 10.0 ** rng.uniform(-3, 0, D.nnz) * (rng.uniform(size=D.nnz) > 0.1)
    D.eliminate_zeros()
    assert orc.is_directed(D)
    cat["directed"] = _laplacian32(D)
    info = {"wide span": wide.data.max() / wide.data.min()}
    return cat, info


@pytest.fixture(scope="module")
def catalogue(gsp):
    import torch
    cat, info = _build_catalogue()
    out = {}
    for name, L in cat.items():
        lmax = 1.01 * float(abs(L.astype(np.float64)).sum(axis=1).max())
        dev = gsp.graphs.DeviceCSR.from_scipy(L, torch.float32, torch.device("cuda"))
        out[name] = (L, dev, lmax)
    return out, info


NAMES = ["nnz%4=0", "nnz%4=1", "nnz%4=2", "nnz%4=3", "isolated runs", "hub", "renumbered",
         "wide weights", "self-loops, normalized", "directed"]


def _empty_tiles(L, R):
    """Start rows of the tiles [k R, (k+1) R) whose CSR slab is empty."""
    ip = L.indptr
    return [k * R for k in range(L.shape[0] // R) if ip[k * R] == ip[(k + 1) * R]]


def test_catalogue_runs_the_paths_it_targets(gsp, catalogue):
    cat, info = catalogue
    for t in range(4):
        L, dev, _ = cat["nnz%%4=%d" % t]
        assert L.nnz % 4 == t and L.shape[0] % 256 == 0      # last tile of every R ends at nnz
        for nsig, ns in ((8, 1), (16, 1), (64, 1), (64, 2), (64, 3), (128, 3)):
            plan = dev.tile_plan(nsig, ns)
            assert plan is not None and plan.rows_per_tile == _default_r(nsig, ns)
        assert {dev.tile_plan(8, 1).rows_per_tile, dev.tile_plan(16, 1).rows_per_tile,
                dev.tile_plan(64, 1).rows_per_tile, dev.tile_plan(64, 2).rows_per_tile,
                dev.tile_plan(64, 3).rows_per_tile} == {256, 128, 64, 32, 16}
    L, dev, _ = cat["isolated runs"]
    for nsig, ns in ((8, 1), (64, 1), (64, 3)):
        R = dev.tile_plan(nsig, ns).rows_per_tile
        empty = _empty_tiles(L, R)
        assert any(s < 600 for s in empty)
        assert any(2100 <= s < 2700 for s in empty)
        assert any(s >= 4200 for s in empty)
        # an empty slab whose offset is not 16-byte aligned borrows entries of earlier rows
        assert any(L.indptr[s] % 4 != 0 for s in empty)
        assert L.indptr[0] % 4 == 0 and L.indptr[600] == 0
    L, dev, _ = cat["hub"]
    assert np.diff(L.indptr).max() >= 3000
    assert set(np.diff(L.indptr)[np.diff(L.indptr) < 100]) <= {2, 3, 4}
    plan = dev.tile_plan(64, 3)
    assert plan is not None and plan.slab_capacity >= 3000 and plan.stages == 2   # 3 cut to 2
    assert dev.tile_plan(128, 16) is not None
    assert info["wide span"] >= 1e6


# ------------------------------------------------------------------------ single steps
def _sentinel(torch, shape, dtype):
    if dtype == torch.float32:
        return torch.full(shape, NAN32, dtype=torch.int32, device="cuda").view(torch.float32)
    return torch.full(shape, NAN64, dtype=torch.int64, device="cuda").view(torch.float64)


def _bits(torch, t):
    return t.view(torch.int32 if t.dtype == torch.float32 else torch.int64).cpu()


def _call_step(dev, plan, first, rb, re, xc, xo, xn, r, r_rows, nsig, ns, ck, c0, a, b, g):
    from pygsp_b200 import _native as nat
    nat.call("gsp_cheby_step_" + nat.suffix(dev.dtype), nat.i32(int(first)), nat.i64(rb),
             nat.i64(re), nat.i64(dev.nnz), dev.indptr, dev.indices, dev.data, xc, xo, xn, r,
             nat.i64(r_rows), nat.i64(nsig), nat.i32(ns), ck, c0, nat.f64(a), nat.f64(b),
             nat.f64(g), plan, nat.stream_ptr(dev.device))


def _check_steps(gsp, L, dev, lmax, nsig, ns, first, plan, seed, label, dtype=np.float32):
    """One step over [0, n) into a fresh buffer, then over [rb, re) with x_new aliasing x_old
    and r_rows > n: in range every element within the bound, out of range bit-unchanged."""
    import torch
    tdt = torch.float32 if dtype == np.float32 else torch.float64
    rng = np.random.default_rng(seed)
    n = L.shape[0]
    xc = so.scaled_signals(rng, n, nsig, dtype)
    xo = so.scaled_signals(rng, n, nsig, dtype)
    rold = np.stack([so.scaled_signals(rng, n, nsig, dtype) for _ in range(max(ns, 1))])
    ck = np.ascontiguousarray(rng.standard_normal(max(ns, 1)))
    c0 = np.ascontiguousarray(rng.standard_normal(max(ns, 1)))
    a, b, g = 3.7 / lmax, -1.93, (0.0 if first else -0.87)
    ref_x, ref_r, bx, br = so.step_reference(L, xc, xo, rold[:ns] if ns else None, a, b, g,
                                             ck, c0, first, dtype)
    xc_d = torch.from_numpy(xc).cuda()
    xo_d = torch.from_numpy(xo).cuda()
    rb = 4 * max(1, (n // 5) // 4)
    re = n - 5
    for lo, hi, alias, r_rows in ((0, n, False, n), (rb, re, not first, n + 12)):
        r_buf = _sentinel(torch, (max(ns, 1), r_rows, nsig), tdt)
        if not first and ns:
            r_buf[:ns, lo:hi] = torch.from_numpy(rold[:ns, lo:hi]).cuda()
        xn = xo_d.clone() if alias else _sentinel(torch, (n, nsig), tdt)
        x_before, r_before = _bits(torch, xn), _bits(torch, r_buf)
        _call_step(dev, plan, first, lo, hi, xc_d, None if first else (xn if alias else xo_d),
                   xn, r_buf, r_rows, nsig, ns, ck, c0, a, b, g)
        torch.cuda.synchronize()
        what = "%s nsig=%d nscales=%d first=%d rows [%d, %d) alias=%d" % (label, nsig, ns, first, lo, hi, alias)
        x_after, r_after = _bits(torch, xn), _bits(torch, r_buf)
        inside = np.zeros(n, dtype=bool)
        inside[lo:hi] = True
        assert torch.equal(x_after[~torch.from_numpy(inside)], x_before[~torch.from_numpy(inside)]), what
        got = xn.cpu().numpy()[lo:hi]
        bad = so.violations(got, ref_x[lo:hi], bx[lo:hi])
        assert not bad.any(), _explain(what + " x_new", bad, got, ref_x[lo:hi], bx[lo:hi], lo)
        rin = np.zeros(r_rows, dtype=bool)
        rin[lo:hi] = True
        mask = torch.from_numpy(np.broadcast_to(rin, (max(ns, 1), r_rows)).copy())
        if ns == 0:
            mask[:] = False
        assert torch.equal(r_after[~mask], r_before[~mask]), what + " (r outside the range)"
        for k in range(ns):
            got = r_buf[k, lo:hi].cpu().numpy()
            bad = so.violations(got, ref_r[k, lo:hi], br[k, lo:hi])
            assert not bad.any(), _explain(what + " r_%d" % k, bad, got, ref_r[k, lo:hi], br[k, lo:hi], lo)


def _explain(what, bad, got, ref, bound, row0):
    i, j = np.argwhere(bad)[0]
    return "%s: %d elements outside the bound, first row %d col %d: got %r ref %r bound %.3g" % (
        what, int(bad.sum()), row0 + i, j, float(got[i, j]), float(ref[i, j]), float(bound[i, j]))


@pytest.mark.parametrize("name", NAMES)
def test_single_steps_within_the_bound(gsp, catalogue, monkeypatch, name):
    cat, _ = catalogue
    L, dev, lmax = cat[name]
    tiled = 0
    for nsig in NSIGS:
        for ns in NSCALES:
            for p2 in (("0", "1") if nsig >= 32 else ("1",)):
                monkeypatch.setenv("GSPB200_TILE_P2", p2)
                plan = dev.tile_plan(nsig, ns)
                tiled += plan is not None
                for first in (True, False):
                    _check_steps(gsp, L, dev, lmax, nsig, ns, first, plan,
                                 seed=nsig * 100 + ns, label="%s P2=%s" % (name, p2))
    assert tiled >= 30                      # most (nsig, nscales) pairs run the tiled kernel


@pytest.mark.parametrize("name", ["isolated runs", "hub", "wide weights", "self-loops, normalized", "directed"])
def test_float64_steps_within_the_bound(gsp, catalogue, name):
    import torch
    cat, _ = catalogue
    L, _, lmax = cat[name]
    dev = gsp.graphs.DeviceCSR.from_scipy(L.astype(np.float64), torch.float64, torch.device("cuda"))
    assert dev.tile_plan(8, 1) is None                # float64 always takes the row-group kernel
    for nsig in (1, 3, 5, 200):
        for ns in ((0, 2, 16) if nsig < 200 else (0, 2)):
            for first in (True, False):
                _check_steps(gsp, L.astype(np.float64), dev, lmax, nsig, ns, first, None,
                             seed=nsig + ns, label=name + " f64", dtype=np.float64)


@pytest.mark.parametrize("nsig,ns", [(8, 1), (64, 1), (64, 3), (128, 2)])
def test_graphs_of_about_one_tile(gsp, monkeypatch, nsig, ns):
    """n < R (no plan), n = R (one tile), n = R + 1..3 (one tile + rows on the row-group kernel)."""
    import torch
    R = _default_r(nsig, ns)
    for n in (R - 4, R, R + 1, R + 2, R + 3):
        L = _laplacian32(so.sensor_adjacency(n, k=6, seed=n))
        lmax = 1.01 * float(abs(L.astype(np.float64)).sum(axis=1).max())
        dev = gsp.graphs.DeviceCSR.from_scipy(L, torch.float32, torch.device("cuda"))
        plan = dev.tile_plan(nsig, ns)
        assert (plan is None) == (n < R)
        assert plan is None or plan.rows_per_tile == R
        for first in (True, False):
            _check_steps(gsp, L, dev, lmax, nsig, ns, first, plan, seed=n, label="n=%d" % n)
        _whole_calls(gsp, L, dev, lmax, nsig, ns, monkeypatch, seed=n, order=7)


# ------------------------------------------------------------------------ whole calls
def _coeffs(rng, rows, order):
    return rng.standard_normal((rows, order + 1)) / np.arange(1, order + 2) ** 2


def _run_forms(gsp, dev, lmax, c_fwd, c_cl, x, src):
    import torch
    from pygsp_b200.filters import approximations as apx
    fwd = apx.cheby_op_device(dev, lmax, c_fwd, x)
    cl = apx.cheby_clenshaw_device(dev, lmax, c_cl, src)
    torch.cuda.synchronize()
    return fwd.clone(), cl.clone()


VARIANTS = ([{"GSPB200_TILE_P2": p, "GSPB200_TILE_VDIR": v} for p in "01" for v in "01"]
            + [{"GSPB200_TILE_S": s} for s in "234"]
            + [{"GSPB200_TILE_NW": w} for w in ("1", "3", "8", "16")]
            + [{"GSPB200_TILE_BPS": "1"}, {"GSPB200_TILE_BPS": "0"},
               {"GSPB200_TILE_HINT": "0"}, {"GSPB200_TILE_HINT": "1"},
               {"GSPB200_TILE_REV": "0"}, {"GSPB200_TILE_REV": "1"},
               {"GSPB200_TILE_SMEM": "8192"}, {"GSPB200_TILE_R": "8"}, {"GSPB200_TILE_R": "24"},
               {"GSPB200_FORCE_HALO": "1"}, {"GSPB200_KERNEL": "rowgroup"}])


def _variants_agree(gsp, dev, lmax, nsig, ns, monkeypatch, c_fwd, c_cl, x, src, variants):
    """(forward, clenshaw) of the default launch, after checking that every variant (plan cache
    cleared for each setting) gives the same bits."""
    base = None
    for env in [{}] + list(variants):
        with monkeypatch.context() as m:
            for k, v in env.items():
                m.setenv(k, v)
            dev._plans.clear()
            plan = dev.tile_plan(nsig, ns)
            if "GSPB200_KERNEL" in env:
                assert plan is None
            elif "GSPB200_TILE_R" in env and plan is not None:
                assert plan.rows_per_tile == max(8, (int(env["GSPB200_TILE_R"]) // (2 if nsig == 128 else 1)) // 8 * 8)
            elif "GSPB200_TILE_S" in env and plan is not None:
                assert plan.stages <= int(env["GSPB200_TILE_S"])
            fwd, cl = _run_forms(gsp, dev, lmax, c_fwd, c_cl, x, src)
        dev._plans.clear()
        if base is None:
            base = (fwd, cl)
            continue
        what = "nsig=%d nscales=%d %s" % (nsig, ns, env)
        assert _same(fwd, base[0]), ("forward form differs", what, _ndiff(fwd, base[0]))
        assert _same(cl, base[1]), ("Clenshaw form differs", what, _ndiff(cl, base[1]))
        del fwd, cl
    return base


def _same(a, b):
    import torch
    return a.shape == b.shape and bool(torch.equal(a, b))


def _ndiff(a, b):
    d = (a != b)
    return int(d.sum()), float((a - b).abs().max() / b.abs().max())


def _whole_calls(gsp, L, dev, lmax, nsig, ns, monkeypatch, seed, order=12, variants=VARIANTS,
                 oracle_cols=None):
    """Forward (ns filters) and Clenshaw (ns sources) calls: identical bits across every launch
    variant and the row-group kernel, and within 1e-5 of the float64 oracle."""
    import torch
    rng = np.random.default_rng(seed)
    n = L.shape[0]
    nf = max(ns, 1)
    x = torch.from_numpy(so.scaled_signals(rng, n, nsig)).cuda()
    src = torch.from_numpy(np.stack([so.scaled_signals(rng, n, nsig) for _ in range(nf)])).cuda()
    c_fwd, c_cl = _coeffs(rng, nf, order), _coeffs(rng, nf, order)
    fwd, cl = _variants_agree(gsp, dev, lmax, nsig, nf, monkeypatch, c_fwd, c_cl, x, src, variants)
    cols = slice(None) if oracle_cols is None else slice(0, oracle_cols)
    Lo = L.astype(np.float64)
    xh = x[:, cols].double().cpu().numpy()
    ref = orc.cheby_op(Lo, lmax, c_fwd, xh)
    assert relerr_cols(fwd[:, :, cols].reshape(nf * n, -1).cpu().numpy(), ref) <= F32_TOL
    refc = sum(orc.cheby_op(Lo, lmax, c_cl[i], src[i][:, cols].double().cpu().numpy())
               for i in range(nf))
    assert relerr_cols(cl[:, cols].cpu().numpy(), refc) <= F32_TOL


@pytest.mark.parametrize("name", NAMES)
def test_whole_calls_and_launch_variants(gsp, catalogue, monkeypatch, name):
    cat, _ = catalogue
    L, dev, lmax = cat[name]
    for nsig, ns in ((8, 1), (16, 2), (32, 3), (64, 1), (64, 5), (128, 2), (64, 16)):
        _whole_calls(gsp, L, dev, lmax, nsig, ns, monkeypatch, seed=nsig + ns)


@pytest.mark.parametrize("name", ["nnz%4=1", "isolated runs", "hub", "wide weights"])
def test_clenshaw_orders_and_sources(gsp, catalogue, name):
    """cheby_clenshaw_device with 1, 2, 5 and 16 sources at orders 1, 2, 3 and 30."""
    import torch
    from pygsp_b200.filters import approximations as apx
    cat, _ = catalogue
    L, dev, lmax = cat[name]
    Lo = L.astype(np.float64)
    rng = np.random.default_rng(31)
    for nsrc, nsig in ((1, 64), (2, 16), (5, 32), (16, 8)):
        src = torch.from_numpy(np.stack([so.scaled_signals(rng, L.shape[0], nsig) for _ in range(nsrc)])).cuda()
        for order in (1, 2, 3, 30):
            c = _coeffs(rng, nsrc, order)
            got = apx.cheby_clenshaw_device(dev, lmax, c, src).cpu().numpy()
            ref = sum(orc.cheby_op(Lo, lmax, c[i], src[i].double().cpu().numpy()) for i in range(nsrc))
            assert relerr_cols(got, ref) <= F32_TOL, (nsrc, order)


# --------------------------------------------------------------- ring wrap-around (2^18 rows)
@pytest.fixture(scope="module")
def big(gsp):
    G = gsp.graphs.Sensor(1 << 18, k=8, seed=7, order="morton")
    G.estimate_lmax()
    return G


def _rounds_ok(torch, plan, n, nsig, bps):
    """n_tiles >= (2 stages + 1) x SMs x CTAs/SM: every CTA passes its ring's parity flip at
    least twice.  CTAs/SM is bounded by the threads a CTA takes (1 + consumer warps)."""
    props = torch.cuda.get_device_properties(0)
    warps = plan.consumer_warps if nsig < 32 else min(plan.consumer_warps, 8)
    per_sm = props.max_threads_per_multi_processor // (32 * (1 + warps))
    if bps:
        per_sm = min(per_sm, bps)
    n_tiles = n // plan.rows_per_tile
    return n_tiles >= (2 * plan.stages + 1) * props.multi_processor_count * per_sm, n_tiles


WRAP = [(16, 1, 0), (32, 2, 0), (64, 2, 0), (64, 3, 0), (128, 3, 0), (64, 16, 0),
        (8, 1, 1), (64, 1, 1), (128, 1, 1), (64, 2, 1)]


@pytest.mark.parametrize("nsig,ns,bps", WRAP)
def test_ring_wraps_and_steps_stay_exact(gsp, big, monkeypatch, nsig, ns, bps):
    import torch
    dev = big.L
    n = dev.shape[0]
    if bps:
        monkeypatch.setenv("GSPB200_TILE_BPS", "1")
    dev._plans.clear()
    plan = dev.tile_plan(nsig, ns)
    assert plan is not None and plan.rows_per_tile == _default_r(nsig, ns)
    assert plan.blocks_per_sm == bps
    ok, n_tiles = _rounds_ok(torch, plan, n, nsig, bps)
    assert ok, (n_tiles, plan.as_dict())
    assert n % plan.rows_per_tile == 0                   # the last tile ends at nnz
    if (nsig, ns, bps) in ((16, 1, 0), (32, 2, 0), (64, 2, 0), (64, 1, 1)):
        L = dev.to_scipy()
        for first in ((True, False) if nsig == 16 else (False,)):
            _check_steps(gsp, L, dev, big.lmax, nsig, ns, first, plan, seed=nsig + ns,
                         label="2^18 rows bps=%d" % bps)
    dev._plans.clear()


@pytest.mark.parametrize("nsig,ns", [(16, 1), (64, 2), (64, 3), (128, 3)])
def test_ring_wrap_whole_calls(gsp, big, monkeypatch, nsig, ns):
    """All launch variants give the same bits at 2^18 rows; two columns against the oracle."""
    variants = [v for v in VARIANTS if "GSPB200_TILE_R" not in v] + [{"GSPB200_TILE_R": "24"}]
    _whole_calls(gsp, big.L.to_scipy(), big.L, big.lmax, nsig, ns, monkeypatch, seed=ns,
                 order=30, variants=variants, oracle_cols=2)
