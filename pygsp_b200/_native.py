"""ctypes binding of libgspb200.so (the C ABI declared in include/gspb200.h).

There is NO fallback: if the shared library cannot be built or loaded, or no
CUDA device is present when a kernel is requested, the call raises.
"""
import ctypes
import os
import re

import numpy as np

from . import build as _build

_HERE = os.path.dirname(os.path.abspath(__file__))
_HEADER = os.path.join(os.path.dirname(_HERE), "include", "gspb200.h")
_lib = None


class NativeError(RuntimeError):
    pass


class TilePlan(ctypes.Structure):
    """Mirror of ``gsp_tile_plan`` (include/gspb200.h)."""
    _fields_ = [("rows_per_tile", ctypes.c_int), ("slab_capacity", ctypes.c_int),
                ("stages", ctypes.c_int), ("consumer_warps", ctypes.c_int),
                ("gather_unroll", ctypes.c_int), ("blocks_per_sm", ctypes.c_int)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class RingPlan(ctypes.Structure):
    """Mirror of ``gsp_ring_plan`` (include/gspb200.h)."""
    _fields_ = [("rows_per_tile", ctypes.c_int), ("ring_max", ctypes.c_int),
                ("tile_meta", ctypes.c_void_p), ("runs", ctypes.c_void_p), ("local", ctypes.c_void_p)]


class HaloFusion(ctypes.Structure):
    """Mirror of ``gsp_halo_fusion`` (include/gspb200.h)."""
    _fields_ = [("n_push_rows", ctypes.c_int64), ("n_push_tiles", ctypes.c_int64),
                ("push_ptr", ctypes.c_void_p), ("push_peer", ctypes.c_void_p),
                ("push_row", ctypes.c_void_p), ("peer_base", ctypes.c_void_p),
                ("peer_flags", ctypes.c_void_p), ("push_counter", ctypes.c_void_p),
                ("wait_flags", ctypes.c_void_p), ("wait_ids", ctypes.c_void_p),
                ("publish_value", ctypes.c_uint64), ("wait_value", ctypes.c_uint64),
                ("n_neighbors", ctypes.c_int32), ("n_wait", ctypes.c_int32),
                ("n_boundary_rows", ctypes.c_int64), ("n_wait_tiles", ctypes.c_int64),
                ("n_owned", ctypes.c_int64), ("publish", ctypes.c_int32),
                ("reserved", ctypes.c_int32)]


class DistPlan(ctypes.Structure):
    """Mirror of ``gsp_dist_plan`` (include/gspb200.h)."""
    _fields_ = [("n_local", ctypes.c_int64), ("n_halo", ctypes.c_int64), ("nnz", ctypes.c_int64),
                ("indptr", ctypes.c_void_p), ("indices", ctypes.c_void_p), ("data", ctypes.c_void_p),
                ("buf", ctypes.c_void_p * 3), ("peer_base", ctypes.c_void_p * 3),
                ("peer_flags", ctypes.c_void_p), ("flags", ctypes.c_void_p),
                ("neighbor_ids", ctypes.c_void_p), ("n_neighbors", ctypes.c_int32),
                ("separate_exchange", ctypes.c_int32), ("push_counter", ctypes.c_void_p),
                ("fused_counter", ctypes.c_void_p), ("n_send", ctypes.c_int64),
                ("src_row", ctypes.c_void_p), ("dst_peer", ctypes.c_void_p),
                ("dst_row", ctypes.c_void_p), ("n_push_rows", ctypes.c_int64),
                ("push_ptr", ctypes.c_void_p), ("push_peer", ctypes.c_void_p),
                ("push_row", ctypes.c_void_p), ("n_boundary_rows", ctypes.c_int64),
                ("perm", ctypes.c_void_p)]


# Scratch of the FISTA solvers (csrc/reduce.cuh): [1] the stop criterion (0 = running), [2] the
# stop iteration, and the history from this offset (GSPB200_FB_HISTORY = GSPB200_TV_HISTORY).
FISTA_HISTORY = 3080


def header_symbols():
    """Every function name include/gspb200.h declares (macro-expanded)."""
    text = open(_HEADER).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    templ, body = [], text
    for macro in re.finditer(r"#define GSPB200_DECLARE_[A-Z]+_API\(SUF, T\)(.*?)\n\n", text, flags=re.S):
        templ += re.findall(r"\b(gsp_[a-z0-9_]+_)##SUF", macro.group(1))
        body = body.replace(macro.group(0), "")
    out = set(re.findall(r"\b(gsp_[a-z0-9_]+)\s*\(", body))
    for t in templ:
        out.add(t + "f32")
        out.add(t + "f64")
    return sorted(out)


def lib():
    """Load (building in-tree if needed) the shared library."""
    global _lib
    if _lib is None:
        # rebuilds only when the sources' hash differs from the one the .so was built from
        path = _build.build(force=bool(os.environ.get("GSPB200_REBUILD")))
        try:
            _lib = ctypes.CDLL(path)
        except OSError as exc:   # pragma: no cover
            raise NativeError("cannot load %s: %s" % (path, exc))
        _lib.gsp_last_error.restype = ctypes.c_char_p
        _lib.gsp_abi_version.restype = ctypes.c_int
        if _lib.gsp_abi_version() != 3:
            raise NativeError("libgspb200 ABI mismatch")
    return _lib


def _arg(a):
    """torch tensor -> device pointer; None -> NULL; numpy -> host pointer."""
    if a is None:
        return ctypes.c_void_p(0)
    if isinstance(a, (TilePlan, RingPlan, HaloFusion, DistPlan)):
        return ctypes.byref(a)
    if hasattr(a, "data_ptr"):
        return ctypes.c_void_p(a.data_ptr())
    if isinstance(a, np.ndarray):
        return ctypes.c_void_p(a.ctypes.data)
    return a


def call(name, *args):
    fn = getattr(lib(), name)
    fn.restype = ctypes.c_int
    rc = fn(*[_arg(a) for a in args])
    if rc != 0:
        msg = lib().gsp_last_error().decode(errors="replace")
        if rc == -1 and "invalid shape" in msg:
            raise TypeError("The coefficients have an invalid shape")
        raise NativeError("%s failed (%d): %s" % (name, rc, msg))


def suffix(dtype):
    import torch
    if dtype in (torch.float32, np.float32) or dtype == np.dtype("float32"):
        return "f32"
    if dtype in (torch.float64, np.float64) or dtype == np.dtype("float64"):
        return "f64"
    raise TypeError("unsupported dtype %r (float32 / float64 only)" % (dtype,))


def i64(v):
    return ctypes.c_int64(int(v))


def i32(v):
    return ctypes.c_int(int(v))


def u64(v):
    return ctypes.c_uint64(int(v))


def f64(v):
    return ctypes.c_double(float(v))


def stream_ptr(device=None):
    import torch
    return ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def require_cuda():
    import torch
    if not torch.cuda.is_available():
        raise NativeError("pygsp_b200 needs a CUDA device (H100): there is no CPU fallback")
    return torch


def run_fista(enqueue, batch, last_pass, width, device, what):
    """Run a FISTA solver to its stop and return ``(scal, niter, crit code, batches)``.

    ``enqueue(it0, it1, cap, scal)`` enqueues passes [it0, it1) on a zero-initialised scratch of
    ``FISTA_HISTORY + width * cap`` doubles (``width`` history entries per pass).  Batches of
    ``batch`` passes alternate with reads of the stop record; the history grows by doubling as the
    run goes on.  ``last_pass`` (None: unbounded) is the pass by which the solver's own rule has
    stopped it, else ``NativeError`` names the solver ``what``.
    """
    torch = require_cuda()
    cap = 1024 if last_pass is None else min(last_pass + 1, 1024)
    scal = torch.zeros(FISTA_HISTORY + width * cap, dtype=torch.float64, device=device)
    done = batches = 0
    while True:
        nxt = done + batch if last_pass is None else min(done + batch, last_pass + 1)
        if nxt > cap:
            cap = max(2 * cap, nxt) if last_pass is None else min(max(2 * cap, nxt), last_pass + 1)
            scal = torch.cat([scal, scal.new_zeros(FISTA_HISTORY + width * cap - scal.numel())])
        enqueue(done, nxt, cap, scal)
        done, batches = nxt, batches + 1
        rec = scal[:3].cpu().numpy()
        if rec[1] != 0:
            return scal, int(rec[2]), int(rec[1]), batches
        if last_pass is not None and done > last_pass:
            raise NativeError("the %s solver did not stop at maxit" % what)
