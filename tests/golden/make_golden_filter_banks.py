"""Generate tests/golden/filter_banks.npz from the unmodified PyGSP 0.6.1 (CPU, NumPy path).

    PYGSP_REFERENCE=<PyGSP 0.6.1 source tree> python tests/golden/make_golden_filter_banks.py

The graph is graphs.Sensor(123, seed=42) of the reference's test_filters.py, the graph of
sensor123.npz (its adjacency is checked against that file), with its full Fourier basis.
Contents (read by tests/test_filter_designs_cpu.py and tests/test_filter_banks_gpu.py):

  lmax, e, U           the reference's G.lmax (= e[-1]), eigenvalues and eigenvectors
  signal               the reference's test_signal: default_rng(42).uniform(size=N)
  grid                 257 frequencies evenly spaced on [0, lmax]
  <d>_grid, <d>_e      evaluate() of design <d> on the grid and at e, (Nf, 257) and (Nf, N)
  <d>_bounds           estimate_frame_bounds() (default x), (2,)
  <d>_cheby, <d>_exact analysis of the signal, method "chebyshev" (order 30) and "exact", (N, Nf)
                       where <d> is every design, with default arguments (name alone) and with
                       one non-default set each (name + "_alt"); see DESIGNS below
  <h>_compl_grid/_e    evaluate() of <h>.complement(2.5) on the grid and at e
  <h>_inv_grid/_e      evaluate() of <h>.inverse() on the grid and at e
                       for h in heat234 (Heat(scale=[2, 3, 4])), abspline5 (Abspline(Nf=5)) and
                       expwin (Expwin()); heat234's complement(2.5) is infeasible (its energy
                       reaches 3) and raises ValueError in the reference, recorded as
                       heat234_compl_raises = 1
  gabor_rect           Gabor(G, Rectangular(G, None, 0.1)).filter(signal), exact, (N, N)
  gabor_delta          Gabor(G, Rectangular(G, 0, 0)).filter(signal), (N, N)
  mod_first_delta      Modulation(G, Rectangular(G, 0, 0), modulation_first=True).filter(signal)
  mod_first_rect       Modulation(G, Rectangular(G, None, 0.1), modulation_first=True).filter(signal)
  mod_second_rect      Modulation(G, Rectangular(G, None, 0.1)).filter(signal), (N, N)
The Modulation outputs depend on the signs of the eigenvectors in U (stored alongside).
"""
import logging
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("PYGSP_REFERENCE") or (sys.argv[1] if len(sys.argv) > 1 else None)
OUT = os.path.join(HERE, "filter_banks.npz")

# name -> (class name, default kwargs, non-default kwargs)
DESIGNS = {
    "abspline": ("Abspline", {}, dict(Nf=4, lpfactor=10)),
    "expwin": ("Expwin", {}, dict(band_min=0.1, band_max=0.7, slope=3)),
    "halfcosine": ("HalfCosine", {}, dict(Nf=4)),
    "held": ("Held", {}, dict(a=0.5)),
    "itersine": ("Itersine", {}, dict(Nf=8, overlap=3)),
    "meyer": ("Meyer", {}, dict(Nf=4)),
    "papadakis": ("Papadakis", {}, dict(a=0.5)),
    "rectangular": ("Rectangular", {}, dict(band_min=0.3, band_max=0.6)),
    "regular": ("Regular", {}, dict(degree=5)),
    "simoncelli": ("Simoncelli", {}, dict(a=0.5)),
    "simpletight": ("SimpleTight", {}, dict(Nf=4)),
    "wave": ("Wave", {}, dict(time=[5, 15], speed=[0.5, 1.5])),
}


def main():
    if not REF:
        raise SystemExit(__doc__)
    sys.path.insert(0, REF)
    from pygsp import filters, graphs
    logging.disable(logging.CRITICAL)
    out = {}
    G = graphs.Sensor(123, seed=42)
    G.compute_fourier_basis()
    ref = np.load(os.path.join(HERE, "sensor123.npz"))
    W = G.W.tocsr()
    assert np.array_equal(W.indptr, ref["W_indptr"]) and np.array_equal(W.indices, ref["W_indices"])
    assert np.array_equal(W.data, ref["W_data"])
    out["lmax"] = np.float64(G.lmax)
    out["e"], out["U"] = G.e, G.U
    signal = np.random.default_rng(42).uniform(size=G.N)
    out["signal"] = signal
    grid = np.linspace(0, G.lmax, 257)
    out["grid"] = grid

    for name, (cls, default, alt) in DESIGNS.items():
        for key, kwargs in ((name, default), (name + "_alt", alt)):
            f = getattr(filters, cls)(G, **kwargs)
            out[key + "_grid"] = f.evaluate(grid)
            out[key + "_e"] = f.evaluate(G.e)
            out[key + "_bounds"] = np.array(f.estimate_frame_bounds())
            out[key + "_cheby"] = f.filter(signal, method="chebyshev", order=30).reshape(G.N, -1)
            out[key + "_exact"] = f.filter(signal, method="exact").reshape(G.N, -1)

    banks = {"heat234": filters.Heat(G, scale=[2, 3, 4]), "abspline5": filters.Abspline(G, 5),
             "expwin": filters.Expwin(G)}
    for name, g in banks.items():
        c = g.complement(2.5)
        try:
            out[name + "_compl_grid"] = c.evaluate(grid)
            out[name + "_compl_e"] = c.evaluate(G.e)
        except ValueError:
            out[name + "_compl_raises"] = np.int64(1)
        h = g.inverse()
        out[name + "_inv_grid"] = h.evaluate(grid)
        out[name + "_inv_e"] = h.evaluate(G.e)

    rect = filters.Rectangular(G, None, 0.1)
    delta = filters.Rectangular(G, 0, 0)
    out["gabor_rect"] = filters.Gabor(G, rect).filter(signal)
    out["gabor_delta"] = filters.Gabor(G, delta).filter(signal)
    out["mod_first_delta"] = filters.Modulation(G, delta, modulation_first=True).filter(signal)
    out["mod_first_rect"] = filters.Modulation(G, rect, modulation_first=True).filter(signal)
    out["mod_second_rect"] = filters.Modulation(G, rect).filter(signal)

    np.savez_compressed(OUT, **out)
    print("wrote", OUT, len(out), "arrays")


if __name__ == "__main__":
    main()
