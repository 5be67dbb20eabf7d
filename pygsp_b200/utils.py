"""Host utilities of the filtering path (mirror of the used part of pygsp/utils.py)."""
import functools
import logging

import numpy as np
from scipy import sparse


def build_logger(name):
    """Per-module logger with the reference's format (pygsp/utils.py:16-31)."""
    logger = logging.getLogger(name)
    if not logger.handlers:
        handler = logging.StreamHandler()
        handler.setLevel(logging.DEBUG)
        handler.setFormatter(logging.Formatter(
            "%(asctime)s:[%(levelname)s](%(name)s.%(funcName)s): %(message)s"))
        logger.setLevel(logging.DEBUG)
        logger.addHandler(handler)
    return logger


def filterbank_handler(func):
    """Call ``func`` once per filter of a bank (pygsp/utils.py:37-53).

    With ``i=`` given, or a single filter, the call goes straight through;
    otherwise the results for i = 0..Nf-1 are collected in a list.
    """
    @functools.wraps(func)
    def wrapper(f, *args, **kwargs):
        if "i" in kwargs or f.Nf <= 1:
            return func(f, *args, **kwargs)
        return [func(f, *args, i=i, **kwargs) for i in range(f.Nf)]
    return wrapper


def compute_log_scales(lmin, lmax, Nscales, t1=1, t2=2):
    """Log-spaced wavelet scales from t2/lmin down to t1/lmax (pygsp/utils.py:312-339)."""
    return np.exp(np.linspace(np.log(t2 / lmin), np.log(t1 / lmax), Nscales))


def resistance_distance(G):
    r"""Resistance distances of a graph (pygsp/utils.py:140-181): a dense (N, N) float64 ndarray.

    ``G``: a :class:`pygsp_b200.graphs.Graph` with a combinatorial Laplacian (else
    ``ValueError``) or a Laplacian as a sparse matrix.  Computed on the device from one float64
    Cholesky factor (:func:`pygsp_b200.reduction.resistance_distance`).
    """
    from .reduction import resistance_distance as _device_resistance_distance
    return _device_resistance_distance(G)


def symmetrize(W, method="average"):
    """Host-side symmetrisation used by the graph generators (pygsp/utils.py:184-277).

    'average' ((W+W^T)/2), 'maximum', 'fill' (fill the zeros of each triangle from the
    other, then average) and 'tril' / 'triu' (mirror one triangle).
    """
    if W.shape[0] != W.shape[1]:
        raise ValueError("Matrix must be square.")
    if method == "average":
        return (W + W.T) / 2
    if method == "maximum":
        if sparse.issparse(W):
            return W.maximum(W.T)
        return np.maximum(W, W.T)
    if method == "fill":
        A = W > 0
        if sparse.issparse(W):
            W = W + ((A + A.T) - A).multiply(W.T)
        else:
            W = W + np.logical_xor(np.logical_or(A, A.T), A) * W.T
        return symmetrize(W, "average")
    if method in ("tril", "triu"):
        tri = getattr(sparse if sparse.issparse(W) else np, method)(W)
        return symmetrize(tri, "maximum")
    raise ValueError("Unknown symmetrization method {}.".format(method))


def bind_to_gpu_numa(device_index=0):
    """Pin this process (and the host memory it allocates from now on) to the NUMA node of a GPU.

    One process per GPU: the pinned staging buffers of Filter.filter's host path should
    live on the socket the GPU hangs off, otherwise every transfer crosses the inter-socket
    link (on an 8-GPU box half of the ranks do by default).  Uses NVML's ideal-CPU mask of
    the device (matched by UUID, so CUDA_VISIBLE_DEVICES renumbering is harmless) and the
    first-touch policy.  Returns the number of CPUs in the mask, or 0 when NVML is not usable
    (nothing is changed then).
    """
    import os
    try:
        import pynvml
        import torch
        pynvml.nvmlInit()
        uuid = str(torch.cuda.get_device_properties(device_index).uuid)
        if not uuid.startswith("GPU-"):
            uuid = "GPU-" + uuid
        handle = pynvml.nvmlDeviceGetHandleByUUID(uuid.encode() if hasattr(uuid, "encode") else uuid)
        words = (os.cpu_count() + 63) // 64
        mask = pynvml.nvmlDeviceGetCpuAffinity(handle, words)
        cpus = [64 * w + b for w, m in enumerate(mask) for b in range(64) if (int(m) >> b) & 1]
        allowed = sorted(set(cpus) & set(os.sched_getaffinity(0)))
        if not allowed:
            return 0
        os.sched_setaffinity(0, allowed)
        return len(allowed)
    except Exception:
        return 0
