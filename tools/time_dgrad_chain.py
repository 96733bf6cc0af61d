#!/usr/bin/env python
"""Device time of the trunk backward's input gradients alone (width 256, 8 layers, skip at 4: layers 6 ... 1, 3-pass
bf16 halves as tc_3x runs them): the fused dgrad_chain_kernel against the layer-by-layer input-gradient GEMMs, both
through sparf_tc_selftest_dgrad_chain, so each call also packs the input gradient's image and the weight images (the
same work in both) and allocates its scratch on the stream.
CUDA events around N calls after a warm-up; the two variants alternate, best of three rounds.  Printed per case: ms per
call, the HBM bytes the variant must move (counted from the shapes: the fp32 input gradient read and its image written;
then per layer the mask bits, the transposed image out and, layer by layer, the row image in and out; the fused chain
reads the first row image once and writes the row images of G[skip] and G[0]) over that time, and the 3-pass tensor
FLOP/s (3 x 2 x rows x 256 x 256 per layer).  Bounds (H100 SXM data sheet): 3.35 TB/s HBM, 989 TFLOP/s dense bf16.
Usage: python tools/time_dgrad_chain.py [calls]"""
import ctypes
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

from sparf_b200 import _lib

W, NT, SKIP, E3 = 256, 8, 4, 63
LAYERS = NT - 2
HBM_PEAK, TENSOR_PEAK = 3.35e12, 989e12


def _p(t):
    return ctypes.c_void_p(t.data_ptr())


def bytes_per_row(chain):
    img = W * 2 * 2                                    # one row of an image, hi and lo halves
    n = 4 * W + img                                    # the input gradient: fp32 read, image written
    per_layer = W / 8 + img                            # mask bits in, transposed image out
    if chain:
        return n + img + LAYERS * per_layer + 2 * img  # its image read once; the row images of G[skip] and G[0]
    return n + LAYERS * (per_layer + 2 * img)          # every layer reads its input's row image and writes its output's


def main():
    calls = int(sys.argv[1]) if len(sys.argv) > 1 else 30
    if not torch.cuda.is_available():
        sys.exit("time_dgrad_chain: needs a GPU")
    print("device: %s; %s" % (torch.cuda.get_device_name(0), subprocess.run(
        ["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
        text=True).stdout.strip()))
    L = _lib.lib()
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    g = torch.Generator(device="cpu").manual_seed(0)
    ks = [(E3 if l == 0 else W) + (E3 if l == SKIP else 0) for l in range(NT)]
    w = torch.cat([(torch.randn(W, k, generator=g) * (2.0 / k) ** 0.5).reshape(-1) for k in ks]).cuda()
    flop_row = 3 * 2 * W * W * LAYERS
    for M in (131072, 65536):
        G = torch.randn(M, W, generator=g).cuda()
        bits = torch.randint(-2 ** 31, 2 ** 31, (LAYERS, M, W // 32), generator=g, dtype=torch.int64).to(torch.int32).cuda()
        tr = torch.empty(LAYERS * 2 * -(-M // 32) * 8192, dtype=torch.int16, device="cuda")
        row = torch.empty(2 * -(-M // 128) * 8 * 8192, dtype=torch.int16, device="cuda")
        db = torch.empty(LAYERS, W, device="cuda")

        def run(chain):
            _lib.check(L.sparf_tc_selftest_dgrad_chain(_p(G), M, E3, NT, SKIP, _p(w), _p(bits), 3, 3, 0, chain, ctypes.c_void_p(0),
                                                       _p(tr), _p(row), _p(db), st), "tc_selftest_dgrad_chain")

        ms = {0: [], 1: []}
        for rep in range(4):                        # the first round is the warm-up
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
            b = M * bytes_per_row(chain)
            print("rows %6d %-14s %.3f ms/call (runs: %s)  %.2f GB -> %.0f GB/s = %.0f %% of HBM peak;  %.0f TFLOP/s 3-pass = "
                  "%.0f %% of tensor peak" % (M, "fused chain" if chain else "layer by layer", t * 1e3,
                                              " ".join("%.3f" % x for x in ms[chain]), b / 1e9, b / t / 1e9,
                                              100 * b / t / HBM_PEAK, M * flop_row / t / 1e12, 100 * M * flop_row / t / TENSOR_PEAK))


if __name__ == "__main__":
    main()
