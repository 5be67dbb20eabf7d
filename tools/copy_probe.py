"""PCIe staging rates of column chunks of a row-major pinned (n, 64) float32 block (needs a GPU).

    python tools/copy_probe.py [--n 1000000]

For chunk widths of 16 / 32 / 64 signals (64 / 128 / 256 contiguous bytes per row, host pitch
256 B): host->device and device->host by the copy engines (cudaMemcpy2DAsync) and by the
zero-copy kernel (gsp_stage_cols) at several grid sizes, each alone, then both directions at
once.  One JSON line per measurement (GB/s of payload).
"""
import argparse
import ctypes
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    a = ap.parse_args()
    import torch
    from pygsp_b200 import _native as nat
    from pygsp_b200 import utils
    utils.bind_to_gpu_numa(0)
    n, nsig, item = a.n, 64, 4
    xh = torch.empty((n, nsig), dtype=torch.float32).pin_memory()
    xh.normal_()
    yh = torch.empty((n, nsig), dtype=torch.float32).pin_memory()
    dev = torch.device("cuda:0")
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()

    def copy(dst, dp, src, sp, w, kind, stream, blocks):
        if blocks:
            nat.call("gsp_stage_cols", ctypes.c_void_p(dst), ctypes.c_size_t(dp), ctypes.c_void_p(src),
                     ctypes.c_size_t(sp), ctypes.c_size_t(w), ctypes.c_size_t(n), nat.i32(blocks),
                     ctypes.c_void_p(stream.cuda_stream))
        else:
            nat.call("gsp_copy2d_async", ctypes.c_void_p(dst), ctypes.c_size_t(dp), ctypes.c_void_p(src),
                     ctypes.c_size_t(sp), ctypes.c_size_t(w), ctypes.c_size_t(n), nat.i32(kind),
                     ctypes.c_void_p(stream.cuda_stream))

    def timed(fn, reps=5):
        import time
        fn()
        torch.cuda.synchronize()
        best = 1e9
        for _ in range(reps):
            torch.cuda.synchronize()
            w0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            best = min(best, time.perf_counter() - w0)
        return best

    for cols in (16, 32, 64):
        w = cols * item
        d = torch.empty((n, cols), dtype=torch.float32, device=dev)
        d2 = torch.randn((n, cols), dtype=torch.float32, device=dev)
        payload = n * w / 1e9
        for blocks in (0, 16, 64, 296):
            how = "dma" if blocks == 0 else "kernel_%d_blocks" % blocks
            t_up = timed(lambda: copy(d.data_ptr(), w, xh.data_ptr(), nsig * item, w, 1, s1, blocks))
            t_dn = timed(lambda: copy(yh.data_ptr(), nsig * item, d2.data_ptr(), w, w, 2, s2, blocks))

            def both():
                copy(d.data_ptr(), w, xh.data_ptr(), nsig * item, w, 1, s1, blocks)
                copy(yh.data_ptr(), nsig * item, d2.data_ptr(), w, w, 2, s2, blocks)
            t_both = timed(both)
            print(json.dumps({"cols": cols, "row_bytes": w, "how": how, "h2d_GBps": payload / t_up,
                              "d2h_GBps": payload / t_dn, "both_GBps_each": payload / t_both,
                              "h2d_ms": 1e3 * t_up, "d2h_ms": 1e3 * t_dn, "both_ms": 1e3 * t_both}))
            sys.stdout.flush()
    # contiguous reference: the whole block each way
    d = torch.empty((n, nsig), dtype=torch.float32, device=dev)
    t_up = timed(lambda: d.copy_(xh, non_blocking=True))
    t_dn = timed(lambda: yh.copy_(d, non_blocking=True))
    print(json.dumps({"cols": 64, "how": "torch copy_ contiguous", "h2d_GBps": n * 256 / 1e9 / t_up,
                      "d2h_GBps": n * 256 / 1e9 / t_dn}))


if __name__ == "__main__":
    main()
