#!/usr/bin/env python
"""Device time of the trunk forward alone (width 256, 8 layers, skip at 4, 3-pass fp16 halves as tc_3x runs it): the fused
trunk_chain_kernel against the layer-by-layer GEMMs, both through sparf_tc_selftest_chain, so each call also packs the
encoding image and the weight images (the same work in both) and allocates its scratch on the stream.
CUDA events around N calls after a warm-up; the two variants alternate.  Printed per case: ms per call, the HBM bytes
the variant must move (counted from the shapes: encoding fp32 in and image out and in, fp32 activations kept, row images
written and read) over that time, and the 3-pass tensor FLOP/s (3 x 2 x rows x sum of K x 256).  Bounds (H100 SXM data
sheet): 3.35 TB/s HBM, 989 TFLOP/s dense fp16.
Usage: python tools/time_trunk_chain.py [calls]"""
import ctypes
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

from sparf_b200 import _lib

W, NT, SKIP, E3, E3P = 256, 8, 4, 63, 64
HBM_PEAK, TENSOR_PEAK = 3.35e12, 989e12


def _p(t):
    return ctypes.c_void_p(t.data_ptr())


def bytes_per_row(chain, taped):
    img = lambda cols: cols * 2 * 2                    # hi and lo halves
    n = 4 * E3P + 2 * img(E3P)                         # the encoding: fp32 read, image written, image read
    kept = NT if taped else 2
    if chain:
        return n + 4 * W * kept + img(W)               # fp32 activations kept, the last row image
    n += img(E3P)                                      # read again at the skip layer
    return n + NT * (4 * W + img(W)) + (NT - 1) * img(W)   # every layer writes fp32 and its image; the next reads it


def main():
    calls = int(sys.argv[1]) if len(sys.argv) > 1 else 30
    if not torch.cuda.is_available():
        sys.exit("time_trunk_chain: needs a GPU")
    print("device: %s; %s" % (torch.cuda.get_device_name(0), subprocess.run(
        ["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
        text=True).stdout.strip()))
    L = _lib.lib()
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    g = torch.Generator(device="cpu").manual_seed(0)
    ks = [(E3 if l == 0 else W) + (E3 if l == SKIP else 0) for l in range(NT)]
    w = torch.cat([(torch.randn(W, k, generator=g) * (2.0 / k) ** 0.5).reshape(-1) for k in ks]).cuda()
    bias = (torch.randn(NT, W, generator=g) * 0.1).cuda()
    flop_row = 3 * 2 * W * sum(-(-k // 32) * 32 for k in ks)
    for M in (131072, 65536):
        enc = torch.zeros(M, E3P)
        enc[:, :E3] = torch.randn(M, E3, generator=g)
        enc = enc.cuda()
        H = torch.empty(NT, M, W, device="cuda")
        last = torch.empty(-(-M // 128) * 8 * 8192, dtype=torch.int16, device="cuda")
        for taped in (True, False):
            outputs = (1 << NT) - 1 if taped else 3 << (NT - 2)

            def run(chain):
                _lib.check(L.sparf_tc_selftest_chain(_p(enc), M, E3, NT, SKIP, _p(w), _p(bias), 3, 1, 0, chain, outputs,
                                                     ctypes.c_void_p(0), _p(H), _p(last), st), "tc_selftest_chain")

            ms = {0: [], 1: []}
            for rep in range(4):                    # the first round is the warm-up
                for chain in (0, 1):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(calls):
                        run(chain)
                    e1.record()
                    torch.cuda.synchronize()
                    if rep:
                        ms[chain].append(e0.elapsed_time(e1) / calls)
            for chain in (0, 1):
                t = min(ms[chain]) * 1e-3
                b = M * bytes_per_row(chain, taped)
                print("rows %6d %-7s %-14s %.3f ms/call (runs: %s)  %.2f GB -> %.0f GB/s = %.0f %% of HBM peak;  %.0f TFLOP/s "
                      "3-pass = %.0f %% of tensor peak" % (M, "taped" if taped else "untaped", "fused chain" if chain else "layer by layer",
                                                           t * 1e3, " ".join("%.3f" % x for x in ms[chain]), b / 1e9, b / t / 1e9,
                                                           100 * b / t / HBM_PEAK, M * flop_row / t / 1e12,
                                                           100 * M * flop_row / t / TENSOR_PEAK))


if __name__ == "__main__":
    main()
