import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def load_golden(name):
    return dict(np.load(os.path.join(GOLDEN, name + ".npz"), allow_pickle=False))


def csr_from(gold, prefix):
    from scipy import sparse
    shape = tuple(int(v) for v in gold[prefix + "_shape"])
    return sparse.csr_matrix((gold[prefix + "_data"], gold[prefix + "_indices"],
                              gold[prefix + "_indptr"]), shape=shape)


@pytest.fixture(scope="session")
def golden():
    cache = {}

    def get(name):
        if name not in cache:
            cache[name] = load_golden(name)
        return cache[name]
    return get


def relerr_cols(y, ref):
    """Parity metric of SURVEY.md 8c: per output column max|y-ref| / max|ref|."""
    y = np.asarray(y, dtype=np.float64).reshape(ref.shape[0], -1)
    r = np.asarray(ref, dtype=np.float64).reshape(ref.shape[0], -1)
    den = np.maximum(np.abs(r).max(axis=0), 1e-300)
    return float((np.abs(y - r).max(axis=0) / den).max())
