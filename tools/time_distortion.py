#!/usr/bin/env python
"""Time the distortion regulariser's fused forward + backward (sparf_distortion_fwd_bwd: d_t's memset and
distortion_kernel).  Prints one JSON line with the device name and power limit.

    python tools/time_distortion.py [--rays 4096] [--samples 128 256] [--calls 200]

For each S: R rays of S samples (t sorted uniform in [2, 6], w = rand^3).  Kernel times: --calls calls of the C ABI on
preallocated buffers (d_t's memset and the kernel, or the kernel alone without d_t) captured in one CUDA graph, CUDA
events around 10 replays, the median of 5 such runs: a Python launch costs more than the kernel at these sizes.  Op
time: the same around eager calls of ops.distortion_loss + backward (allocation, autograd and launches included).
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch

from sparf_b200 import _lib, ops
from time_density import power_limit


def time_calls(fn, calls, runs=5):
    """Median over runs of the microseconds per call of `fn`, called `calls` times between two events."""
    for _ in range(3):
        fn()
    out = []
    for _ in range(runs):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(calls):
            fn()
        e1.record()
        torch.cuda.synchronize()
        out.append(e0.elapsed_time(e1) * 1e3 / calls)
    return statistics.median(out)


def time_graphed(fn, calls, replays=10):
    """Microseconds per call of `fn` from replays of one CUDA graph holding `calls` calls."""
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        fn()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(calls):
            fn()
    return time_calls(graph.replay, replays) / calls


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rays", type=int, default=4096)
    ap.add_argument("--samples", type=int, nargs="+", default=[128, 256])
    ap.add_argument("--calls", type=int, default=200)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "time_distortion.py measures on a GPU"
    L = _lib.lib()
    out = dict(device=torch.cuda.get_device_name(), power_limit_w=power_limit(), rays=args.rays,
               lib=os.path.basename(os.environ.get("SPARF_B200_LIB", "")) or "libsparf_b200.so", us={})
    g = torch.Generator(device="cuda").manual_seed(0)
    for S in args.samples:
        R = args.rays
        t = torch.sort(torch.rand(R, S, device="cuda", generator=g) * 4 + 2, dim=1).values
        w = torch.rand(R, S, device="cuda", generator=g) ** 3
        loss, d_w, d_t = torch.zeros((), device="cuda"), torch.empty_like(w), torch.empty_like(t)

        def kernel(d_t):
            _lib.check(L.sparf_distortion_fwd_bwd(R, S, ops._ptr(t), ops._ptr(w), 1.0, ops._ptr(loss), ops._ptr(d_w),
                                                  ops._ptr(d_t), ops._stream()), "distortion")

        tg, wg = t[..., None].clone().requires_grad_(True), w[..., None].clone().requires_grad_(True)

        def op():
            ops.distortion_loss(tg, wg).backward()

        out["us"]["S%d" % S] = dict(kernel_with_d_t=round(time_graphed(lambda: kernel(d_t), args.calls), 2),
                                    kernel_without_d_t=round(time_graphed(lambda: kernel(None), args.calls), 2),
                                    op_fwd_bwd=round(time_calls(op, args.calls), 2))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
