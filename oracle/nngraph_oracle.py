"""Float64 restatement of NNGraph, ImgPatches and Grid2dImgPatches
(pygsp/graphs/nngraphs/nngraph.py:92-299, imgpatches.py:51-105, grid2dimgpatches.py:37-43) and of
utils.symmetrize (pygsp/utils.py:244-277), held to tests/golden/nngraph.npz.

Host only and direct on purpose: scipy's cKDTree for the searches, the reference's sparse
formulas for the symmetrisations, numpy's sliding windows for the patches.  It shares no code
with the device engine (pygsp_b200/graphs/generators.py, csrc/neighbors.cu), which the GPU tests
hold to the same fixture.
"""
import numpy as np
from scipy import sparse, spatial

DIST_ORDER = {"euclidean": 2.0, "manhattan": 1.0, "max_dist": np.inf}


def symmetrize(W, method):
    """utils.symmetrize of a sparse matrix, formula for formula."""
    if method == "average":
        return (W + W.T) / 2
    if method == "maximum":
        bigger = W.T > W
        return W - W.multiply(bigger) + W.T.multiply(bigger)
    if method == "fill":
        A = W > 0
        mask = (A + A.T) - A
        return symmetrize(W + mask.multiply(W.T), "average")
    if method in ("tril", "triu"):
        return symmetrize(getattr(sparse, method)(W), "maximum")
    raise ValueError(method)


def prepare(Xin, center=True, rescale=True):
    """nngraph.py:127-136."""
    X = np.array(Xin, dtype=np.float64)
    N, d = X.shape
    if center:
        X = X - X.mean(axis=0)
    if rescale:
        radius = 0.5 * np.linalg.norm(X.max(axis=0) - X.min(axis=0), 2)
        X *= (np.power(N, 1.0 / float(min(d, 3))) / 10.0) / radius
    return X


def minkowski(u, v, p):
    """scipy.spatial.distance.minkowski (what nngraph.py:243 calls)."""
    return np.linalg.norm(u - v, ord=p)


def nngraph(Xin, NNtype="knn", k=10, epsilon=0.01, p=2.0, symmetrize_type="average"):
    """(W as canonical CSR, sigma) of NNGraph(Xin, ...) with the default center / rescale."""
    X = prepare(Xin)
    N = X.shape[0]
    tree = spatial.cKDTree(X)
    if NNtype == "knn":
        D, NN = tree.query(X, k=k + 1, p=p)
        sigma = np.mean(D[:, 1:])
        rows = np.repeat(np.arange(N), k)
        cols, dist = NN[:, 1:].ravel(), D[:, 1:].ravel()
    else:
        rows, cols, dist = [], [], []
        for i in range(N):
            for j in tree.query_ball_point(X[i], r=epsilon, p=p):
                if j != i:
                    rows.append(i)
                    cols.append(j)
                    dist.append(minkowski(X[i], X[j], p))
        if not dist:
            raise ValueError("No neighbors found")
        rows, cols, dist = np.array(rows), np.array(cols), np.array(dist)
        sigma = np.mean(dist)
    W = sparse.csc_matrix((np.exp(-dist ** 2 / float(sigma)), (rows, cols)), shape=(N, N))
    W = sparse.csr_matrix(symmetrize(W, symmetrize_type))
    W.eliminate_zeros()
    W.sort_indices()
    return W, sigma


def patches(img, patch_shape):
    """Feature rows of ImgPatches: symmetric padding, one r x c (x C) window per pixel."""
    img = np.asarray(img, dtype=np.float64)
    h, w = img.shape[:2]
    r = patch_shape[0]
    c = patch_shape[1] if len(patch_shape) > 1 else r
    pad = [(int((r - 0.5) / 2.0), int((r + 0.5) / 2.0)), (int((c - 0.5) / 2.0), int((c + 0.5) / 2.0))]
    if img.ndim == 3:
        pad.append((0, 0))
    P = np.pad(img, pad, mode="symmetric")
    if img.ndim == 2:
        P = P[:, :, None]
    win = np.lib.stride_tricks.sliding_window_view(P, (r, c), axis=(0, 1))   # (h, w, C, r, c)
    return np.ascontiguousarray(win.transpose(0, 1, 3, 4, 2)).reshape(h * w, -1)


def grid2d(h, w):
    """Adjacency of Grid2d(h, w) (grid2d.py:40-89): 4 neighbours, unit weights, row-major."""
    N = h * w
    right = np.ones(N - 1)
    right[w - 1::w] = 0
    W = sparse.diags([right, np.ones(N - w)], [1, w], shape=(N, N), format="csr")
    W.eliminate_zeros()
    return (W + W.T).tocsr()


def img_patches(img, patch_shape):
    return nngraph(patches(img, patch_shape))


def grid2d_img_patches(img, patch_shape):
    Wp, sigma = img_patches(img, patch_shape)
    W = (Wp + grid2d(img.shape[0], img.shape[1])).tocsr()
    W.sort_indices()
    return W, sigma
