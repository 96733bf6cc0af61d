#!/usr/bin/env python
"""Kernel time of one weight-gradient GEMM dW[N x K] += G^T X over M = 131 072 rows (a c2 chunk) at the shapes of the
network: K = 256 (trunk layers, the colour head's features), 64 (the position encoding), 32 with one row per 128 rows
(the direction encoding); N = 256 (trunk) and 128 (colour head).  Two paths on the same values:
  staged: X with 16-byte aligned rows, split inside the GEMM (wg_gemm_staged_kernel);
  packed: X copied to rows of K + 1 floats, which the bulk copies cannot read: pack_kernel<TnB> + wg_gemm_kernel.
Device time per call from torch.profiler over repeated calls after a warm-up (sparf_tc_selftest_wgrad; its transposed
image of G and its memsets are not counted).  Beside the times, each shape's bounds from the data sheet of the H100 SXM:
  HBM: the transposed image of G (2 bytes per value and pass, N padded to 128-row tiles) and X in fp32, at 3.35 TB/s;
  MMA: the products of the passes at 989 dense bf16 TFLOP/s, N x K per row with K padded to the 128-wide B tile (the
  products the GEMM issues; K = 64 and 32 half- or quarter-fill it).
Usage: [SPARF_TW_PASSES=3|1] python tools/time_wgrad.py [calls]"""
import ctypes
import os
import subprocess
import sys
from collections import defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from torch.profiler import ProfilerActivity, profile

from sparf_b200 import _lib

M = 131072
HBM_PEAK = 3.35e12      # H100 SXM data sheet, bytes/s
MMA_PEAK = 989e12       # dense bf16 FLOP/s, same source
SHAPES = [(256, 256, 1), (256, 128, 1), (64, 256, 1), (64, 128, 1), (32, 256, 128), (32, 128, 128)]   # K, N, div


def main():
    calls = int(sys.argv[1]) if len(sys.argv) > 1 else 20
    passes = int(os.environ.get("SPARF_TW_PASSES", "3"))
    if not torch.cuda.is_available():
        sys.exit("time_wgrad: needs a GPU")
    L = _lib.lib()
    p = torch.cuda.get_device_properties(0)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print("device: %s, %d SMs (%s); M = %d, %d passes, %d calls per path" % (p.name, p.multi_processor_count, smi, M,
                                                                           passes, calls))
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    g = torch.Generator(device="cuda").manual_seed(0)
    print("%5s %5s %5s | %8s %8s | %10s %10s %10s | %10s | %6s" % ("K", "N", "div", "HBM us", "MMA us", "pack us",
                                                                     "gemm us", "sum us", "staged us", "ratio"))
    for K, N, div in SHAPES:
        rows = -(-M // div)
        hbm = (M * -(-N // 128) * 128 * 2 * (2 if passes == 3 else 1) + rows * K * 4) / HBM_PEAK * 1e6
        mma = passes * 2.0 * M * N * -(-K // 128) * 128 / MMA_PEAK * 1e6
        G = torch.randn(M, N, device="cuda", generator=g)
        X = torch.randn(rows, K, device="cuda", generator=g)
        Xodd = torch.empty(rows, K + 1, device="cuda")
        Xodd[:, :K] = X
        dW = torch.empty(N, K, device="cuda")
        bits = torch.empty(M, -(-K // 32), dtype=torch.int32, device="cuda")

        def run(x, ldx):
            _lib.check(L.sparf_tc_selftest_wgrad(ctypes.c_void_p(G.data_ptr()), ctypes.c_void_p(x.data_ptr()), M, N, K,
                                                 K, ldx, div, passes, 0, ctypes.c_void_p(dW.data_ptr()),
                                                 ctypes.c_void_p(bits.data_ptr()), stream), "tc_selftest_wgrad")

        t = defaultdict(float)
        for x, ldx in ((X, K), (Xodd, K + 1)):
            for _ in range(3):
                run(x, ldx)
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(calls):
                    run(x, ldx)
                torch.cuda.synchronize()
            for ev in prof.events():
                if ev.device_type.name != "CUDA":
                    continue
                if "wg_gemm_staged_kernel" in ev.name:
                    t["staged"] += ev.device_time / calls
                elif "wg_gemm_kernel" in ev.name:
                    t["gemm"] += ev.device_time / calls
                elif "pack_kernel" in ev.name and "TnB" in ev.name:
                    t["pack"] += ev.device_time / calls
        packed = t["pack"] + t["gemm"]
        print("%5d %5d %5d | %8.1f %8.1f | %10.1f %10.1f %10.1f | %10.1f | %6.3f" % (
            K, N, div, hbm, mma, t["pack"], t["gemm"], packed, t["staged"], t["staged"] / packed))


if __name__ == "__main__":
    main()
