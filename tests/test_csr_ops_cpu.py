"""CSR structure on the device has one owner, checked without a GPU: only graphs/csr.py calls the
native entry points that assemble, transpose, symmetrise, compact or slice a CSR matrix, and
``DeviceCSR.from_coo`` refuses 2^31 triplets before it converts, allocates or needs a device."""
import os
import re

import pytest

PKG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "pygsp_b200")
OWNER = os.path.join("graphs", "csr.py")
STRUCTURE_CALLS = re.compile(r"gsp_coo_to_csr|gsp_csr_transpose|gsp_csr_average_|"
                             r"gsp_csr_symmetrize_|gsp_csr_compact_|gsp_vertex_map|gsp_subgraph_")


def _sources():
    for root, _, files in os.walk(PKG):
        for name in sorted(files):
            if name.endswith(".py"):
                path = os.path.join(root, name)
                with open(path, encoding="utf-8") as fh:
                    yield os.path.relpath(path, PKG), fh.read()


def test_only_csr_module_builds_csr_structure():
    offenders = [(name, m.group(0)) for name, text in _sources() if name != OWNER
                 for m in STRUCTURE_CALLS.finditer(text)]
    assert offenders == []


def test_from_coo_refuses_2_to_the_31_triplets_first():
    torch = pytest.importorskip("torch")
    from pygsp_b200.graphs.csr import DeviceCSR
    n = 2 ** 31
    rows = torch.empty(n, dtype=torch.int64, device="meta")
    vals = torch.empty(n, dtype=torch.float32, device="meta")
    with pytest.raises(ValueError, match="at most 2\\^31 - 1"):
        DeviceCSR.from_coo(rows, rows, vals, (1000, 1000))
