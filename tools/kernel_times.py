#!/usr/bin/env python
"""Per-kernel device time of one MLP training step / inference forward (torch.profiler = CUPTI activity records, no
replay, warm caches), and the achieved HBM bandwidth of the wgmma GEMM kernels against the bytes they must move.
Usage: [SPARF_KT_ENGINE=tc_3x|tc_1x|tc_3x_w1] [SPARF_KT_NOPOSE=1] python tools/kernel_times.py [R S]"""
import os
import sys
from collections import defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "golden")):
    sys.path.insert(0, p)
import torch
from torch.profiler import ProfilerActivity, profile

import common
from sparf_b200 import _lib, ops

HBM_PEAK = 3.35e12      # H100 SXM data sheet, bytes/s
GEMM_KERNELS = ("wg_gemm_kernel", "wg_gemm_staged_kernel", "trunk_chain_kernel", "dgrad_chain_kernel")
# 16-bit passes of the images (forward, input gradient, weight gradient) per tensor-core engine
PASSES = {"tc_3x": (3, 3, 3), "tc_1x": (1, 1, 1), "tc_3x_w1": (3, 3, 1), "auto": (3, 3, 3)}


def gemm_bytes_per_row(spec, passes, backward, pose):
    """HBM bytes per sample row that the wgmma GEMMs must read and write, counted from the shapes: the A operand images,
    the weight-gradient GEMMs' B operands (the activations, read as fp32 and split inside the GEMM), the fp32 outputs,
    the epilogue images and the ReLU masks (bits, 1/8 byte per value, written by the weight-gradient GEMM; fp32 at the
    last trunk layer, whose epilogue sums the density row's weight gradient from the values; with the fused trunk, the
    masks of H[0] ... H[nt-3] are written by the forward and read by the fused input gradients).  The weights' images are
    small and stay in L2; they are not counted."""
    pf, pd, pw = passes
    W, HW, skip, nt = spec.width, spec.head_width, spec.skip_layer, spec.n_trunk
    E3p, Evp = -(-(3 + 6 * spec.L_xyz) // 8) * 8, -(-(3 + 6 * spec.L_view) // 8) * 8

    def img(cols, p):     # one row of an image: K padded to 32, 2 bytes per half, hi and lo halves when p == 3
        return -(-cols // 32) * 32 * 2 * (2 if p == 3 else 1)

    # forward: the fused trunk (width 256, as MLPSpec's default) reads the encoding image once, keeps the activations on
    # the SM, and writes fp32 H[l] where it is kept (every layer for the tape; the last two in an inference forward) and
    # the last layer's row image; other widths go layer by layer, each reading its input image (+ enc at the skip layer)
    # and writing fp32 H and its row image; a training forward through the fused trunk also writes the masks of H[0] ...
    # H[nt-3].  The colour head reads [H | denc] and writes fp32 hid
    chained = W == 256 and E3p <= 64 and nt >= 3
    if chained:
        n = img(E3p, pf) + 4 * W * (nt if backward else 2) + img(W, pf) + (W / 8 * (nt - 2) if backward else 0)
    else:
        n = sum(img(W if l else E3p, pf) + (img(E3p, pf) if l == skip else 0) + 4 * W + img(W, pf) for l in range(nt))
    n += img(W, pf) + img(Evp, pf) + 4 * HW
    if not backward:
        return n
    # colour head: two weight-gradient GEMMs (Ghid^T [feat | denc]); the input gradient of feat (mask = feat) as row and
    # transposed images; with pose gradients the direction-encoding gradient in fp32
    n += 2 * img(HW, pw) + 4 * W + 4 * Evp
    n += img(HW, pd) + W / 8 + img(W, pd) + img(W, pw)
    if pose:
        n += img(HW, pd) + 4 * Evp
    for l in range(nt - 1, -1, -1):
        n += img(W, pw) + 4 * (W if l else E3p)                         # weight gradient
        if l == skip:
            n += img(W, pw) + 4 * E3p
        if l > 0 and chained and l < nt - 1:
            # the fused input gradients of layers nt-2 ... 1: G[nt-2]'s row image once, per layer the mask and the
            # transposed image out, and the row images of G[skip] and G[0] for the encoding's gradient
            n += (img(W, pd) if l == nt - 2 else 0) + W / 8 + img(W, pw) + (img(W, pd) if pose and (l - 1 in (skip, 0)) else 0)
        elif l > 0:                                                     # input gradient: G image, mask, two images out
            n += img(W, pd) + (4 * W if l == nt - 1 else W / 8) + img(W, pd) + img(W, pw)
        if pose and (l == skip or l == 0):                              # encoding gradient, fp32 (+= at layer 0)
            n += img(W, pd) + 4 * E3p + (4 * E3p if l == 0 and skip > 0 else 0)
    return n


def main():
    R, S = (int(sys.argv[1]), int(sys.argv[2])) if len(sys.argv) > 2 else (1023, 128)
    opt = common.make_opt(S=S)
    sd = common.det_weights(opt, 0)
    keys = sum([["mlp_feat.%d.weight" % i, "mlp_feat.%d.bias" % i] for i in range(8)], []) + \
        ["mlp_rgb.0.weight", "mlp_rgb.0.bias", "mlp_rgb.1.weight", "mlp_rgb.1.bias"]
    params = [sd[k].cuda().requires_grad_(True) for k in keys]
    pose = os.environ.get("SPARF_KT_NOPOSE", "0") != "1"      # ray gradients (camera-pose optimisation) on / off
    o = (torch.randn(R, 3, device="cuda") * 0.3).requires_grad_(pose)
    d = torch.nn.functional.normalize(torch.randn(R, 3, device="cuda"), dim=-1).requires_grad_(pose)
    t = torch.sort(torch.rand(R, S, device="cuda") * 4 + 1.2, dim=1).values
    spec = ops.MLPSpec()
    eng_name = os.environ.get("SPARF_KT_ENGINE", "tc_3x")
    eng = _lib.ENGINES[eng_name]
    gs, gc = torch.randn(R, S, device="cuda"), torch.randn(R, S, 3, device="cuda")

    def step():
        for p in params:
            p.grad = None
        s, c = ops.mlp_forward(spec, o, d, t, params, engine=eng)
        torch.autograd.backward([s, c], [gs, gc])

    def infer():
        with torch.no_grad():
            ops.mlp_forward(spec, o, d, t, params, engine=eng)

    if torch.cuda.is_available():
        p = torch.cuda.get_device_properties(0)
        print("device: %s, %d SMs" % (p.name, p.multi_processor_count))
    for name, fn, bwd in (("training step (forward with tape + backward)", step, True), ("inference forward", infer, False)):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        n = 5
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(n):
                fn()
            torch.cuda.synchronize()
        agg = defaultdict(lambda: [0, 0.0])
        for ev in prof.events():
            if ev.device_type.name == "CUDA":
                agg[ev.name][0] += 1
                agg[ev.name][1] += ev.device_time
        tot = sum(v[1] for v in agg.values()) / n
        print("== %s: %.1f us of kernels per call" % (name, tot))
        for k, v in sorted(agg.items(), key=lambda kv: -kv[1][1]):
            print("  %8.1f us  x%-3d %s" % (v[1] / n, v[0] // n, k[:110]))
        if eng_name in PASSES:
            g_us = sum(v[1] for k, v in agg.items() if any(g in k for g in GEMM_KERNELS)) / n
            g_bytes = R * S * gemm_bytes_per_row(spec, PASSES[eng_name], bwd, pose and bwd)
            print("  GEMM group (%s): %.1f us per call, %.2f GB to move (from shapes), %.0f GB/s = %.1f %% of %.2f TB/s"
                  % (" + ".join(GEMM_KERNELS), g_us, g_bytes / 1e9, g_bytes / (g_us * 1e-6) / 1e9 if g_us else 0.0,
                     100 * g_bytes / (g_us * 1e-6) / HBM_PEAK if g_us else 0.0, HBM_PEAK / 1e12))


if __name__ == "__main__":
    main()
