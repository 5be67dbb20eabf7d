"""Host side of the sampled models (pygsp_b200/graphs/sampled.py) against the PyGSP 0.6.1
fixture tests/golden/sampled_models.npz: coordinates and Community's info bit for bit, argument
errors, and utils.rescale_center / utils.distanz.  No GPU needed."""
import hashlib
import json

import numpy as np
import pytest

from pygsp_b200 import utils
from pygsp_b200.graphs import sampled

GOLD = "sampled_models"


def _digest(a):
    """The fixture's SHA-256 of a float64 array's C-order bytes."""
    return hashlib.sha256(np.ascontiguousarray(a, dtype=np.float64).tobytes()).hexdigest()


def _same(a, g, key):
    assert _digest(a) == str(g[key]), key


def _cases(golden, model):
    g = golden(GOLD)
    return [(str(c), json.loads(str(g[str(c) + "_args"]))["kwargs"]) for c in g["cases"]
            if json.loads(str(g[str(c) + "_args"]))["model"] == model]


def _community_host(N=256, Nc=None, min_comm=None, comm_sizes=None, size_ratio=1, seed=None,
                    **_):
    """The host half of Community.__init__ (labels, info, coordinates, key)."""
    if Nc is None:
        Nc = int(round(np.sqrt(N) / 2))
    if min_comm is None:
        min_comm = int(round(N / (3 * Nc)))
    rng = np.random.default_rng(seed)
    if comm_sizes is None:
        node_com = np.sort(np.concatenate((np.tile(np.arange(Nc), (min_comm,)),
                                           rng.choice(Nc, N - min_comm * Nc))))
    else:
        node_com = np.concatenate([[v] * c for v, c in enumerate(comm_sizes)])
    sizes = np.bincount(node_com, minlength=Nc)
    world_rad = size_ratio * np.sqrt(N)
    com_coords, coords = sampled.community_coordinates(node_com, sizes, world_rad, rng)
    return dict(node_com=node_com, comm_sizes=sizes, world_rad=world_rad,
                com_coords=com_coords), coords


def test_community_coordinates_and_info_bit_equal(golden):
    g = golden(GOLD)
    cases = _cases(golden, "Community")
    assert len(cases) >= 8
    for name, kwargs in cases:
        info, coords = _community_host(**kwargs)
        _same(coords, g, name + "_coords_sha256")
        for key in ("node_com", "comm_sizes", "world_rad", "com_coords"):
            np.testing.assert_array_equal(info[key], g["%s_info_%s" % (name, key)],
                                          err_msg=name + " " + key)


@pytest.mark.parametrize("seed", [0, 1, 2, 3, 4])
def test_community_polar_map_matches_the_reference_loop(seed):
    """The vectorised polar map and offset give the bits of community.py's per-vertex loop."""
    N, Nc = 5000, 35
    rng = np.random.default_rng(seed)
    node_com = np.sort(rng.integers(0, Nc, N))
    sizes = np.bincount(node_com, minlength=Nc)
    world_rad = np.sqrt(N)
    _, coords = sampled.community_coordinates(node_com, sizes, world_rad,
                                              np.random.default_rng(seed + 100))
    com = world_rad * np.array(list(zip(np.cos(2 * np.pi * np.arange(1, Nc + 1) / Nc),
                                        np.sin(2 * np.pi * np.arange(1, Nc + 1) / Nc))))
    ref = np.random.default_rng(seed + 100).uniform(size=(N, 2))
    ref = np.array([[e[0] * np.cos(2 * np.pi * e[1]), e[0] * np.sin(2 * np.pi * e[1])]
                    for e in ref])
    for i in range(N):
        ref[i] = com[node_com[i]] + np.sqrt(sizes[node_com[i]]) * ref[i]
    np.testing.assert_array_equal(coords, ref)


def test_swissroll_points_bit_equal(golden):
    g = golden(GOLD)
    cases = _cases(golden, "SwissRoll")
    assert len(cases) == 6
    for name, kw in cases:
        x = sampled.swissroll_points(kw.get("N", 400), 1, 4, kw.get("dim", 3),
                                     kw.get("noise", False), kw.get("srtype", "uniform"),
                                     kw.get("seed"))
        _same(x, g, name + "_x_sha256")
        _same(utils.rescale_center(x).T, g, name + "_coords_sha256")


def test_swissroll_restatement_gives_the_reference_weights(golden):
    """oracle.swissroll_reference reproduces the reference's weights: the fixture's structure
    exactly and the SHA-256 of its weights (which the fixture keeps instead of the weights)."""
    from oracle import sampled_models_oracle as smo
    g = golden(GOLD)
    for name, kw in _cases(golden, "SwissRoll"):
        N = kw.get("N", 400)
        x = sampled.swissroll_points(N, 1, 4, kw.get("dim", 3), kw.get("noise", False),
                                     kw.get("srtype", "uniform"), kw.get("seed"))
        T = smo.swissroll_reference(utils.rescale_center(x).T, np.sqrt(2.0 / N), 1e-6)
        np.testing.assert_array_equal(T.indptr, g[name + "_W_indptr"], err_msg=name)
        np.testing.assert_array_equal(T.indices, g[name + "_W_indices"], err_msg=name)
        _same(T.data, g, name + "_W_sha256")


def test_sphere_cube_twomoons_points_bit_equal(golden):
    g = golden(GOLD)
    for name, kw in _cases(golden, "Sphere"):
        pts = sampled.sphere_points(kw.get("nb_pts", 300), kw.get("nb_dim", 3), kw.get("seed"))
        _same(pts, g, name + "_coords_sha256")
    for name, kw in _cases(golden, "Cube"):
        pts = sampled.cube_points(kw.get("nb_pts", 300), kw.get("nb_dim", 3), kw.get("seed"))
        _same(pts, g, name + "_coords_sha256")
    for name, kw in _cases(golden, "TwoMoons"):
        N = kw.get("N", 400)
        moon = sampled.TwoMoons._create_arc_moon
        pts = np.concatenate((moon(N // 2, 0.07, 0.5, 1, kw.get("seed")),
                              moon(N - N // 2, 0.07, 0.5, 2, kw.get("seed"))))
        _same(pts, g, name + "_coords_sha256")
        np.testing.assert_array_equal(np.concatenate((np.zeros(N // 2), np.ones(N - N // 2))),
                                      g[name + "_labels"])


def test_sphere_row_norm_differs_from_axis_norm_somewhere():
    """Why sphere_points keeps the reference's row loop: over a few clouds, norm(axis=1) gives
    different bits for some rows, and the loop is what the reference computes."""
    differs = False
    for seed in range(5):
        raw = np.random.RandomState(seed).normal(0, 1, (5000, 3))
        loop = sampled.sphere_points(5000, 3, seed)
        ref = raw.copy()
        for i in range(ref.shape[0]):
            ref[i] = ref[i] / np.linalg.norm(ref[i])
        np.testing.assert_array_equal(loop, ref)
        differs |= not np.array_equal(raw / np.linalg.norm(raw, axis=1)[:, None], loop)
    assert differs


def test_errors_match_the_reference(golden):
    """Every invalid argument set raises the reference's exception type before any device
    work, so this runs without a GPU."""
    errors = json.loads(str(golden(GOLD)["errors"]))
    assert len(errors) >= 12
    for model, kwargs, exc in errors:
        assert exc is not None
        with pytest.raises(getattr(__builtins__, exc, None) or eval(exc)):
            getattr(sampled, model)(**kwargs)


def test_deliberate_errors():
    with pytest.raises(ValueError):
        sampled.Community(N=100, k_neigh=33)
    with pytest.raises(ValueError):
        sampled.SwissRoll(N=100, dim=4)
    with pytest.raises(ValueError):
        sampled.SwissRoll(N=100, srtype="spiral")
    with pytest.raises(ValueError):
        sampled.Cube(nb_dim=1)
    with pytest.raises(NotImplementedError, match="data file"):
        sampled.TwoMoons()


def test_rescale_center_and_distanz_docstring_examples():
    np.testing.assert_allclose(utils.rescale_center(np.array([[1, 6], [2, 5], [3, 4]])),
                               [[-1.0, 1.0], [-0.6, 0.6], [-0.2, 0.2]])
    x = np.arange(3)
    np.testing.assert_array_equal(utils.distanz(x, x),
                                  [[0.0, 1.0, 2.0], [1.0, 0.0, 1.0], [2.0, 1.0, 0.0]])
    np.testing.assert_array_equal(utils.distanz(x), utils.distanz(x, x))
    a, b = np.ones((2, 4)), np.ones((3, 5))
    assert utils.distanz(a, np.ones((2, 5))).shape == (4, 5)
    with pytest.raises(ValueError):
        utils.distanz(a, b)


def test_inflated_probability():
    assert sampled.inflated_probability(0, 10) == 0.0
    assert sampled.inflated_probability(5, 6) == 1.0
    p = sampled.inflated_probability(500000, 5e11)
    assert 500000 / 5e11 < p < 1.02 * 500000 / 5e11     # a 1.1 % margin at n = 5e5
