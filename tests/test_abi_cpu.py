"""CPU-side checks: the C-ABI library builds, loads and exports every symbol the
header declares; host-side logic that needs no GPU."""
import os

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))


def test_library_exports_every_declared_symbol():
    from pygsp_b200 import _native
    lib = _native.lib()
    names = _native.header_symbols()
    assert len(names) >= 36
    for required in ("gsp_cheby_op_f32", "gsp_cheby_step_f64", "gsp_laplacian_fill_f32",
                     "gsp_lanczos_f32", "gsp_spectral_bounds_f64", "gsp_launch_count"):
        assert required in names
    missing = [n for n in names if not hasattr(lib, n)]
    assert not missing, missing
    assert lib.gsp_abi_version() == 2


def test_fista_history_matches_header():
    """The host reads the FISTA solvers' history at the offset both header macros give."""
    import re
    from pygsp_b200 import _native
    text = open(_native._HEADER).read()
    for macro in ("GSPB200_FB_HISTORY", "GSPB200_TV_HISTORY"):
        value = re.search(r"#define %s (\d+)" % macro, text)
        assert value and int(value.group(1)) == _native.FISTA_HISTORY, macro


def test_no_cpu_fallback():
    """Without a CUDA device the product path must fail loudly, not compute on the CPU."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    import pygsp_b200 as gsp
    with pytest.raises(gsp._native.NativeError):
        gsp.graphs.Graph(np.ones((3, 3)) - np.eye(3))


def test_product_never_imports_oracle():
    """The oracle is test infrastructure: nothing shipped may import, link or open it."""
    import os
    import re
    root = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "pygsp_b200")
    uses = re.compile(r"(from|import)\s+oracle|oracle[/.]\w|liboracle|cheby_oracle|pygsp_oracle")
    for dirpath, _, files in os.walk(root):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                text = open(os.path.join(dirpath, f)).read()
                assert not uses.search(text), os.path.join(dirpath, f)


def test_cheby_coefficients_host(golden):
    """compute_cheby_coeff is host code: check it against the PyGSP goldens."""
    from pygsp_b200 import filters

    class FakeGraph:
        lmax = float(golden("sensor123")["lmax"])
        N = 123

    g = golden("sensor123")
    G = FakeGraph()
    np.testing.assert_allclose(filters.compute_cheby_coeff(filters.Heat(G), m=30),
                               g["heat10_coeff"], rtol=1e-10, atol=1e-14)
    c = filters.compute_cheby_coeff(filters.MexicanHat(G, Nf=5), m=40)
    assert isinstance(c, list) and len(c) == 5
    np.testing.assert_allclose(np.array(c), g["mh5_coeff"], rtol=1e-10, atol=1e-13)
    c = filters.compute_cheby_coeff(filters.Heat(G, scale=[8, 9]), m=30, i=1)
    np.testing.assert_allclose(c, g["heat89_coeff"][1], rtol=1e-10, atol=1e-14)
    f = filters.MexicanHat(G, Nf=5)
    assert f.Nf == 5 and len(f) == 5 and f.shape == (5, 1)
    assert f.evaluate(np.linspace(0, G.lmax, 11)).shape == (5, 11)
    assert "MexicanHat(in=1, out=5" in repr(f)
    with pytest.raises(ValueError):
        filters.MexicanHat(G, Nf=5, scales=[1, 2])


def test_morton_order_is_a_permutation():
    from pygsp_b200.graphs import morton_order
    pts = np.random.default_rng(0).uniform(size=(1000, 2))
    perm = morton_order(pts)
    assert sorted(perm.tolist()) == list(range(1000))
    # neighbours in the order are close in space (vs ~0.52 for a random order)
    d = np.linalg.norm(np.diff(pts[perm], axis=0), axis=1).mean()
    assert d < 0.1
    assert sorted(morton_order(np.random.default_rng(1).uniform(size=(500, 3))).tolist()) == list(range(500))


def test_jackson_coefficients(golden):
    """approximations.py:166-225, golden from PyGSP."""
    from pygsp_b200 import filters
    g = golden("jackson")
    bounds = [float(g["bounds"][0]), float(g["bounds"][1])]
    ch, jch = filters.compute_jackson_cheby_coeff(bounds, list(g["lam"]), int(g["m"]))
    np.testing.assert_allclose(ch, g["ch"], rtol=1e-12, atol=1e-15)
    np.testing.assert_allclose(jch, g["jch"], rtol=1e-12, atol=1e-15)
    assert bounds == [1.0, 4.0]                      # the caller's list is left alone
    with pytest.raises(ValueError):
        filters.compute_jackson_cheby_coeff([1.0, 20.0], [0.0, 13.9], 10)


def test_ritz_check_on_a_host_lanczos():
    """The stopping rule shared by Graph.estimate_lmax and the distributed estimate, driven
    by a NumPy Lanczos on a small Laplacian: stops, and the estimate brackets the truth."""
    from scipy import sparse
    from pygsp_b200.graphs.graph import ritz_check
    rng = np.random.default_rng(0)
    A = sparse.random(400, 400, 0.03, random_state=0, format="csr")
    A = A + A.T
    L = (sparse.diags(np.asarray(A.sum(axis=1)).ravel()) - A).tocsr()
    lam = np.linalg.eigvalsh(L.toarray())[-1]
    v = rng.standard_normal(400); v /= np.linalg.norm(v)
    v_prev, beta_prev, alphas, betas = None, 0.0, [], []
    for j in range(200):
        w = L @ v
        a = float(w @ v); w = w - a * v - (beta_prev * v_prev if v_prev is not None else 0)
        b = float(np.linalg.norm(w)); alphas.append(a); betas.append(b)
        if (j + 1) >= 10 and (j + 1 - 10) % 5 == 0:
            theta, m, stop, ref_rule = ritz_check(np.array(alphas), np.array(betas), 5e-3, False, j + 1 >= 60)
            if stop:
                break
        v_prev, beta_prev, v = v, b, w / b
    assert stop and ref_rule and j + 1 <= 60
    assert lam * (1 - 1e-4) <= theta <= lam * (1 + 1e-12)
    # an exactly invariant start vector: beta_0 = 0 stops at once with the exact eigenvalue
    theta, m, stop, _ = ritz_check(np.array([3.0]), np.array([0.0]), 5e-3, False, False)
    assert stop and m == 1 and theta == 3.0


def test_e2e_chunk_plan(monkeypatch):
    """Column chunks of the pinned-host pipeline (filters/pipeline.py): two halves when the half
    is a width the tiled kernel takes and the block is worth pipelining, else the whole block;
    GSPB200_E2E_CHUNK forces equal chunks."""
    from pygsp_b200.filters import pipeline
    monkeypatch.delenv("GSPB200_E2E_CHUNK", raising=False)
    assert pipeline.chunk_plan(1_000_000, 64, 4) == [(0, 32), (32, 32)]
    assert pipeline.chunk_plan(6_250_000, 128, 4) == [(0, 64), (64, 64)]
    assert pipeline.chunk_plan(1_000_000, 16, 4) == [(0, 8), (8, 8)]
    assert pipeline.chunk_plan(1_000_000, 24, 4) == [(0, 24)]          # 12 is not a tiled width
    assert pipeline.chunk_plan(10_000, 64, 4) == [(0, 64)]             # < 32 MB: not worth it
    assert pipeline.chunk_plan(1_000_000, 1, 4) == [(0, 1)]
    monkeypatch.setenv("GSPB200_E2E_CHUNK", "16")
    assert pipeline.chunk_plan(1_000_000, 64, 4) == [(0, 16), (16, 16), (32, 16), (48, 16)]
    monkeypatch.setenv("GSPB200_E2E_CHUNK", "0")
    assert pipeline.chunk_plan(1_000_000, 64, 4) == [(0, 64)]


def test_header_is_plain_c_and_a_c_host_links(tmp_path):
    """include/gspb200.h is a C header (extern "C" boundary: plain pointers and sizes, no C++ or
    torch types), and examples/c_host.c -- a host written in C -- compiles and links against the
    built library.  (It needs a GPU to run; here it must fail cleanly at its first cudaMalloc.)"""
    import shutil
    import subprocess
    root = os.path.dirname(HERE)
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("no gcc")
    hdr = os.path.join(root, "include", "gspb200.h")
    subprocess.run([gcc, "-std=c99", "-Wall", "-Werror", "-fsyntax-only", "-x", "c", hdr], check=True)
    from pygsp_b200 import build
    lib = build.build()
    cuda_lib = "/usr/local/cuda/lib64"
    if not os.path.exists(os.path.join(cuda_lib, "libcudart.so")):
        pytest.skip("no libcudart to link the example against")
    exe = str(tmp_path / "c_host")
    subprocess.run([gcc, "-std=c99", "-Wall", "-I" + os.path.join(root, "include"),
                    os.path.join(root, "examples", "c_host.c"), "-o", exe,
                    "-L" + os.path.dirname(lib), "-lgspb200", "-L" + cuda_lib, "-lcudart", "-lm",
                    "-Wl,-rpath," + os.path.dirname(lib)], check=True)
    import torch
    if not torch.cuda.is_available():
        out = subprocess.run([exe], capture_output=True, text=True)
        assert out.returncode == 1 and "cudaMalloc failed" in out.stderr
