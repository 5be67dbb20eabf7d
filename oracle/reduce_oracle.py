"""NumPy restatement of the fixed summation order of csrc/reduce.cuh: the row partition of a
column reduction and the order in which the per-row terms of each column are added.

``row_parts(n)`` is the partition; ``column_sums(prod)`` adds the (n, b) float64 terms of every
column in the device's order: within part p, warp w sums rows p chunk + w, p chunk + w + 8, ...
from 0.0; the eight warp sums are added in warp order from 0.0, then the part totals in part
order from 0.0.  NumPy float64 adds round to nearest, as the device's do, so when every term is
exact in float64 (a product of two float32 values, say) the result is the device's bit for bit.
"""
import numpy as np

MAX_PARTS = 264      # kMaxParts
WARPS = 8            # kWarps: warps of a 256-thread CTA
TARGET_ROWS = 1024   # rows per part until MAX_PARTS parts are reached


def ceil_div(a, b):
    return -(-a // b)


def row_parts(n):
    """(used, chunk): part p is rows [p chunk, min(n, (p + 1) chunk)), p < used."""
    parts = max(1, min(ceil_div(n, TARGET_ROWS), MAX_PARTS))
    chunk = ceil_div(n, parts)
    return ceil_div(n, chunk), chunk


def column_sums(prod):
    """Per-column totals of the (n, b) float64 terms ``prod`` in the order of csrc/reduce.cuh."""
    prod = np.asarray(prod, dtype=np.float64)
    if prod.ndim == 1:
        prod = prod[:, None]
    n, b = prod.shape
    used, chunk = row_parts(n)
    steps = ceil_div(chunk, WARPS)
    # each part padded with +0.0 to steps * WARPS rows: adding +0.0 leaves every sum unchanged
    pad = np.zeros((used, steps * WARPS, b))
    for p in range(used):
        rows = prod[p * chunk:min(n, (p + 1) * chunk)]
        pad[p, :rows.shape[0]] = rows
    pad = pad.reshape(used, steps, WARPS, b)          # [p, i, w] = row p chunk + 8 i + w
    acc = np.zeros((used, WARPS, b))
    for i in range(steps):
        acc = acc + pad[:, i]
    part = np.zeros((used, b))
    for w in range(WARPS):
        part = part + acc[:, w]
    tot = np.zeros(b)
    for p in range(used):
        tot = tot + part[p]
    return tot
