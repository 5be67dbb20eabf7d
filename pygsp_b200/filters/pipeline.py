"""Filtering of HOST signal blocks with the PCIe transfers overlapped.

``Filter.filter`` / ``cheby_op`` take and return host arrays in the reference
(pygsp/filters/filter.py:146-328, approximations.py:58-114).  Uploading the block,
running the recurrence and downloading the result one after the other makes the two
transfers longer than the recurrence itself (256 MB each way for config 2).  The
recurrence needs all ROWS of its operand before its first step but its COLUMNS are
independent, so the block is cut into column chunks and three streams run as a
pipeline:

    upload stream   : chunk j+1  host -> HBM   (strided 2-D copy of a pinned block)
    compute stream  : chunk j    K fused recurrence steps
    download stream : chunk j-1  HBM -> host

Only page-locked (pinned) torch tensors take this path -- the copy engines cannot run
asynchronously on pageable memory; NumPy / pageable inputs use one plain copy each way.
"""
import ctypes
import os

import numpy as np

from .. import _native as nat

_TILED_WIDTHS = (128, 64, 32, 16, 8)
_streams = {}
last_trace = None      # GSPB200_E2E_TRACE=1: [(stage, chunk, start_ms, end_ms)] of the last call


def _side_streams(device):
    torch = nat.require_cuda()
    key = (device.type, device.index)
    if key not in _streams:
        _streams[key] = (torch.cuda.Stream(device=device), torch.cuda.Stream(device=device))
    return _streams[key]


def chunk_plan(n, nsig, itemsize):
    """Column chunks [(offset, width), ...] for an (n, nsig) block.

    Two halves: 64 signals -> 32 | 32.  Narrower chunks shorten the first upload and the last
    download, which overlap nothing, but every chunk re-reads the CSR arrays at every order and
    narrow blocks run the recurrence less efficiently -- the pipeline is compute-bound, so
    quarters lose (config 2 on an H100 SXM at 400 W: 32 | 32 -> 25.3 ms, whole block 25.2 ms,
    4 x 16 -> 27.7 ms per call; GSPB200_E2E_TRACE=1 records the timelines).  The width must be one the
    tiled kernel supports; blocks that are small (< 32 MB) or do not split that way are taken
    whole.  GSPB200_E2E_CHUNK=w forces equal chunks of w signals (0 = no pipelining)."""
    env = os.environ.get("GSPB200_E2E_CHUNK")
    if env is not None:
        w = int(env)
        if w > 0 and nsig % w == 0:
            return [(o, w) for o in range(0, nsig, w)]
        return [(0, nsig)]
    h = nsig // 2
    if nsig % 2 == 0 and h in _TILED_WIDTHS and n * nsig * itemsize >= (32 << 20):
        return [(0, h), (h, h)]
    return [(0, nsig)]


def _copy2d(dst_ptr, dpitch, src_ptr, spitch, width, height, kind, stream, use_kernel):
    if use_kernel:
        nat.call("gsp_stage_cols", ctypes.c_void_p(dst_ptr), ctypes.c_size_t(dpitch),
                 ctypes.c_void_p(src_ptr), ctypes.c_size_t(spitch), ctypes.c_size_t(width),
                 ctypes.c_size_t(height), nat.i32(int(os.environ.get("GSPB200_STAGE_BLOCKS", "16"))),
                 ctypes.c_void_p(stream.cuda_stream))
    else:
        nat.call("gsp_copy2d_async", ctypes.c_void_p(dst_ptr), ctypes.c_size_t(dpitch),
                 ctypes.c_void_p(src_ptr), ctypes.c_size_t(spitch), ctypes.c_size_t(width),
                 ctypes.c_size_t(height), nat.i32(kind), ctypes.c_void_p(stream.cuda_stream))


def run_pinned(compute, device, dtype, xh, nscales, out=None, chunks=None):
    """The three-stream pipeline for any column-separable operator.

    ``compute(x_chunk)`` maps an (n, w) device block to an (nscales, n, w) device tensor on the
    current stream (it may return a fresh tensor per call; references are kept until the
    downloads have finished).  ``xh``: contiguous pinned host tensor (n, nsig).  Returns the
    pinned host tensor (nscales, n, nsig), complete on return.  ``chunks``: [(offset, width)]
    (default: :func:`chunk_plan`; callers whose ranks must agree pass it explicitly).
    """
    torch = nat.require_cuda()
    n, nsig = xh.shape
    item = xh.element_size()
    if xh.dtype != dtype or not xh.is_contiguous() or not xh.is_pinned():
        raise ValueError("the pipelined path needs a contiguous pinned host tensor of the engine's dtype")
    if out is None:
        out = torch.empty((nscales, n, nsig), dtype=dtype, pin_memory=True)
    chunks = chunks if chunks else chunk_plan(n, nsig, item)
    nchunks = len(chunks)
    use_kernel = os.environ.get("GSPB200_STAGE", "dma") == "kernel"
    with torch.cuda.device(device):
        main = torch.cuda.current_stream(device)
        s_in, s_out = _side_streams(device)
        xin = [torch.empty((n, w), dtype=dtype, device=device) for _, w in chunks]
        trace = os.environ.get("GSPB200_E2E_TRACE") == "1"
        marks = []

        def mark(stage, j, stream):
            if trace:
                ev = torch.cuda.Event(enable_timing=True)
                ev.record(stream)
                marks.append((stage, j, ev))
        mark("t0", -1, main)
        s_in.wait_stream(main)
        s_out.wait_stream(main)
        ev_in = []
        for j, ((o, w), buf) in enumerate(zip(chunks, xin)):   # uploads run back to back on their stream
            mark("up_begin", j, s_in)
            _copy2d(buf.data_ptr(), w * item, xh.data_ptr() + o * item, nsig * item, w * item, n, 1,
                    s_in, use_kernel)
            ev_in.append(s_in.record_event())
            mark("up_end", j, s_in)
        results = []
        for j, (o, w) in enumerate(chunks):
            main.wait_event(ev_in[j])
            mark("compute_begin", j, main)
            res = compute(xin[j])
            results.append(res)
            mark("compute_end", j, main)
            s_out.wait_event(main.record_event())
            mark("down_begin", j, s_out)
            for i in range(nscales):
                _copy2d(out[i].data_ptr() + o * item, nsig * item, res[i].data_ptr(), w * item,
                        w * item, n, 2, s_out, use_kernel)
            mark("down_end", j, s_out)
        main.wait_stream(s_in)
        main.wait_stream(s_out)
        main.synchronize()                     # a host result must be complete on return
        if trace:
            global last_trace
            t0 = marks[0][2]
            last_trace = [(stage, j, round(t0.elapsed_time(ev), 3)) for stage, j, ev in marks[1:]]
    return out


def filter_pinned(L, lmax, c, xh, clenshaw=True, out=None):
    """r = cheby_op(L, c, x) for a PINNED host block ``xh`` (N, nsig) of ``L.dtype``.

    Returns a pinned host tensor (Nscales, N, nsig) (``out`` if given), complete when the
    function returns.  Single-filter banks use the Clenshaw form when ``clenshaw`` (one pass
    less over the block per order, see ``cheby_clenshaw_device``).
    """
    from . import approximations as apx
    c = np.ascontiguousarray(np.atleast_2d(np.asarray(c, dtype=np.float64)))
    nscales = c.shape[0]
    if nscales == 1 and clenshaw:
        compute = lambda xc: apx.cheby_clenshaw_device(L, lmax, c, xc)[None]
    else:
        compute = lambda xc: apx.cheby_op_device(L, lmax, c, xc)
    return run_pinned(compute, L.device, L.dtype, xh, nscales, out)
