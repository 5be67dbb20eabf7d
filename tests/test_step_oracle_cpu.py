"""The float64 step reference and its error bound (oracle/step_oracle.py), without a GPU.

The bound must let every correct answer through and still be tight enough to catch one wrong
entry of one row: a dropped or doubled neighbour, two columns of a packet swapped, a row taken
from a stale stage, a missing x_old term, an accumulator written into the wrong filter.  The same
holds for the Clenshaw form of the step (source blocks added to x_new, no accumulator), where a
missing source or the source of another order must be caught, and for the per-order sources of
the wide synthesis (mix_reference): a coefficient of order 0 not halved, the orders of another
chunk.
"""
import numpy as np
import pytest

from oracle import pygsp_oracle as orc
from oracle import step_oracle as so

R = 64          # rows per tile of the one-filter plan: the distance of a stale stage


@pytest.fixture(scope="module")
def case():
    """A Morton-numbered sensor graph and one step's inputs (16 signals, 3 filters)."""
    W = so.sensor_adjacency(2048, k=8, seed=3)
    L64 = orc.laplacian(W)
    rng = np.random.default_rng(0)
    lmax = float(abs(L64).sum(axis=1).max())
    coef = dict(alpha=4.0 / lmax, beta=-2.0, gamma=-1.0, ck=[0.3, -0.11, 0.071], c0=[0.9, 0.4, -0.2])
    return L64, rng, coef


CS = [1.0, 0.37, -0.21]     # Clenshaw-form source coefficients


def _inputs(L64, dtype, nsig=16, nscales=3, seed=1):
    rng = np.random.default_rng(seed)
    L = L64.astype(dtype)
    n = L.shape[0]
    xc = so.scaled_signals(rng, n, nsig, dtype)
    xo = so.scaled_signals(rng, n, nsig, dtype)
    r = np.stack([so.scaled_signals(rng, n, nsig, dtype) for _ in range(nscales)])
    return L, xc, xo, r


def _reference(L, xc, xo, r, coef, first, dtype, sources):
    """The plain step (accumulators r), or with ``sources`` the Clenshaw form (r as sources)."""
    if sources:
        return so.step_reference(L, xc, xo, None, first=first, dtype=dtype, sources=r, cs=CS,
                                 **coef)
    return so.step_reference(L, xc, xo, r, first=first, dtype=dtype, **coef)


def _check_rounded_reference(case, dtype, first, sources):
    L64, _, coef = case
    L, xc, xo, r = _inputs(L64, dtype)
    x, rr, bx, br = _reference(L, xc, xo, r, coef, first, dtype, sources)
    assert not so.violations(x.astype(dtype), x, bx).any()
    assert not so.violations(rr.astype(dtype), rr, br).any()
    assert rr.shape[0] == (0 if sources else 3)


def _check_perturbed(case, dtype, first, sources):
    L64, rng, coef = case
    L, xc, xo, r = _inputs(L64, dtype)
    x, rr, bx, br = _reference(L, xc, xo, r, coef, first, dtype, sources)
    work = x.dtype
    for ref, b in ((x, bx), (rr, br)):
        sign = np.where(rng.uniform(size=ref.shape) < 0.5, -1.0, 1.0)
        for frac in (0.5, rng.uniform(0, 0.5, ref.shape)):
            got = ref.astype(dtype).astype(work) + (sign * frac * b).astype(work)
            assert not so.violations(got, ref, b).any()


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("first", [True, False])
def test_rounded_reference_passes(case, dtype, first):
    _check_rounded_reference(case, dtype, first, sources=False)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("first", [True, False])
def test_rounded_reference_with_sources_passes(case, dtype, first):
    _check_rounded_reference(case, dtype, first, sources=True)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("first", [True, False])
def test_perturbed_by_half_the_bound_passes(case, dtype, first):
    _check_perturbed(case, dtype, first, sources=False)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("first", [True, False])
def test_perturbed_with_sources_by_half_the_bound_passes(case, dtype, first):
    _check_perturbed(case, dtype, first, sources=True)


def _scale_entry(L, j, factor):
    M = L.copy()
    M.data[j] = M.data[j] * factor
    return M


def test_sources_leave_the_plain_step_unchanged(case):
    """No source term: the same values and bounds as before the term existed; zero sources
    change the value by nothing and only widen the bound."""
    L64, _, coef = case
    L, xc, xo, r = _inputs(L64, np.float32)
    x, rr, bx, br = so.step_reference(L, xc, xo, r, first=False, dtype=np.float32, **coef)
    x2, rr2, bx2, br2 = so.step_reference(L, xc, xo, r, first=False, dtype=np.float32,
                                          sources=None, cs=None, **coef)
    for a, b in ((x, x2), (rr, rr2), (bx, bx2), (br, br2)):
        assert np.array_equal(a, b)
    xz, _, bz, _ = so.step_reference(L, xc, xo, None, first=False, dtype=np.float32,
                                     sources=np.zeros_like(r), cs=CS, **coef)
    assert np.array_equal(xz, x) and np.all(bz >= bx)
    with pytest.raises(ValueError):
        so.step_reference(L, xc, xo, r, first=False, dtype=np.float32, sources=r, cs=CS, **coef)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_mutations_are_rejected(case, dtype):
    _check_mutations(case, dtype, sources=False)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_mutations_with_sources_are_rejected(case, dtype):
    """The Clenshaw form: the step's mutations, a missing source and the wrong source block."""
    _check_mutations(case, dtype, sources=True)


def _check_mutations(case, dtype, sources):
    L64, _, coef = case
    L, xc, xo, r = _inputs(L64, dtype)
    n, nsig = xc.shape
    x, rr, bx, br = _reference(L, xc, xo, r, coef, False, dtype, sources)
    gx, gr = x.astype(dtype), rr.astype(dtype)
    a = dtype(coef["alpha"])

    # a neighbour whose term |alpha w x| exceeds 10x its row's bound
    row = n // 2 + 5
    lo, hi = L.indptr[row], L.indptr[row + 1]
    terms = np.abs(a * L.data[lo:hi, None].astype(np.float64) * xc[L.indices[lo:hi]])
    j_rel, col = np.unravel_index(np.argmax(terms / bx[row][None, :]), terms.shape)
    assert terms[j_rel, col] > 10 * bx[row, col]

    def rejected(got_x, got_r=gr):
        return so.violations(got_x, x, bx).any() or so.violations(got_r, rr, br).any()

    assert not rejected(gx)
    mutants = {}
    for name, factor in (("dropped", 0.0), ("doubled", 2.0)):
        M = _scale_entry(L, lo + j_rel, factor)
        mx, mr, _, _ = _reference(M, xc, xo, r, coef, False, dtype, sources)
        mutants[name] = (mx.astype(dtype), mr.astype(dtype))
    sw = gx.copy()
    sw[row, [4, 5]] = sw[row, [5, 4]]                 # two columns of one 4-column packet
    mutants["swapped columns"] = (sw, gr)
    stale = gx.copy()
    stale[row] = gx[row - R]                          # a row from the stage R rows earlier
    mutants["stale row"] = (stale, gr)
    no_old = gx.copy()
    no_old[row] = (x[row] - dtype(coef["gamma"]) * xo[row].astype(x.dtype)).astype(dtype)
    mutants["gamma x_old omitted"] = (no_old, gr)
    if sources:
        cs = [dtype(c) for c in CS]
        for name, got in (("source 1 omitted", x[row] - cs[1] * r[1, row].astype(x.dtype)),
                          ("source 2 for source 1", x[row] + cs[1] * (r[2, row].astype(x.dtype)
                                                                      - r[1, row]))):
            mutated = gx.copy()
            mutated[row] = got.astype(dtype)
            mutants[name] = (mutated, gr)
    else:
        shifted = gr.copy()
        shifted[1, row] = gr[0, row]                  # r of filter 0 written into filter 1
        mutants["r into the next filter"] = (gx, shifted)
    for name, (mx, mr) in mutants.items():
        assert rejected(mx, mr), name
        # and only the mutated row is flagged
        bad = so.violations(mx, x, bx).any(axis=1) | so.violations(mr, rr, br).any(axis=(0, 2))
        assert np.flatnonzero(bad).tolist() == [row], name


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_mix_reference_bound(dtype):
    """The per-order sources: the rounded reference and a kernel-order float sum pass, half the
    bound passes, c_f0 not halved and the orders of the previous 32-order chunk are rejected."""
    rng = np.random.default_rng(4)
    nsrc, m, n, nsig = 33, 40, 50, 3
    src = np.stack([so.scaled_signals(rng, n, nsig, dtype) for _ in range(nsrc)])
    c = rng.standard_normal((nsrc, m)) / np.arange(1, m + 1)
    u, b = so.mix_reference(src, c, dtype)
    assert u.shape == b.shape == (m, n, nsig)
    assert not so.violations(u.astype(dtype), u, b).any()
    # the kernel's own order: fma from 0 in increasing f, emulated with one rounding per add
    ch = c.copy()
    ch[:, 0] *= 0.5
    ch = ch.astype(dtype)
    acc = np.zeros((m, n, nsig), dtype=dtype)
    for f in range(nsrc):
        acc = (acc.astype(u.dtype) + ch[f][:, None, None].astype(u.dtype) * src[f]).astype(dtype)
    assert not so.violations(acc, u, b).any()
    sign = np.where(rng.uniform(size=u.shape) < 0.5, -1.0, 1.0)
    assert not so.violations(u.astype(dtype).astype(u.dtype) + (0.5 * sign * b).astype(u.dtype),
                             u, b).any()
    c_full = c.copy()
    c_full[:, 0] *= 2.0                               # order 0 not halved
    u_bad, _ = so.mix_reference(src, c_full, dtype)
    assert so.violations(u_bad.astype(dtype), u, b)[0].all(axis=(0, 1)).any()
    assert not so.violations(u_bad.astype(dtype), u, b)[1:].any()
    shifted = u.copy()
    shifted[32:] = u[:m - 32]                         # chunk 2 read the first chunk's orders
    assert so.violations(shifted.astype(dtype), u, b)[32:].any(axis=(1, 2)).all()


def test_signals_scale_columns_by_powers_of_two():
    x = so.scaled_signals(np.random.default_rng(0), 5, 18, np.float64)
    y = so.scaled_signals(np.random.default_rng(0), 5, 18, np.float64)
    assert np.array_equal(x, y)
    base = np.random.default_rng(0).standard_normal((5, 18))
    ratio = x / base
    assert np.array_equal(ratio[0], 2.0 ** ((np.arange(18) % 9) - 4))


def test_sensor_adjacency_is_a_symmetric_knn_graph():
    W = so.sensor_adjacency(500, k=6, seed=1)
    assert (W != W.T).nnz == 0 and W.diagonal().max() == 0
    assert W.getnnz(axis=1).min() >= 6
    assert 0 < W.data.min() and W.data.max() <= 1
