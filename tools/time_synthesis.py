"""Times Filter.filter synthesis (Nf features -> 1) fused vs reference order (needs a GPU)."""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
import bench  # noqa: E402
import pygsp_b200 as gsp  # noqa: E402

n, nsig, nf, order = 1_000_000, 64, 6, 30
G = gsp.graphs.Graph(bench.host_graph(n, 10, 0))
G.estimate_lmax()
bank = gsp.filters.MexicanHat(G, Nf=nf)
s = torch.randn(n, nsig, nf, device="cuda")
out = {}
for fused in (True, False):
    bank.fused_synthesis = fused
    for _ in range(2):
        y = bank.filter(s, order=order)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(3):
        y = bank.filter(s, order=order)
    e1.record()
    torch.cuda.synchronize()
    out["fused" if fused else "reference_order"] = e0.elapsed_time(e1) / 3
    out["y_fused" if fused else "y_ref"] = y
diff = float((out.pop("y_fused") - out.pop("y_ref")).abs().max() / y.abs().max())
print(json.dumps({"synthesis_ms": out, "rel_diff": diff, "N": n, "nsig": nsig, "Nf": nf, "order": order}))
