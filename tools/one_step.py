#!/usr/bin/env python
"""A few taped MLP training steps at the bench shape (1023 rays x 128 samples), e.g. to run under torch.profiler.
[SPARF_OS_ENGINE=tc_3x|tc_3x_w1] python tools/one_step.py [steps]"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "golden")):
    sys.path.insert(0, p)
import torch

import common
from sparf_b200 import _lib, ops


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 3
    R, S = 1023, 128
    opt = common.make_opt(S=S)
    sd = common.det_weights(opt, 0)
    keys = sum([["mlp_feat.%d.weight" % i, "mlp_feat.%d.bias" % i] for i in range(8)], []) + \
        ["mlp_rgb.0.weight", "mlp_rgb.0.bias", "mlp_rgb.1.weight", "mlp_rgb.1.bias"]
    params = [sd[k].cuda().requires_grad_(True) for k in keys]
    o = torch.randn(R, 3, device="cuda") * 0.3
    d = torch.nn.functional.normalize(torch.randn(R, 3, device="cuda"), dim=-1)
    t = torch.sort(torch.rand(R, S, device="cuda") * 4 + 1.2, dim=1).values
    spec = ops.MLPSpec()
    gs, gc = torch.randn(R, S, device="cuda"), torch.randn(R, S, 3, device="cuda")
    for _ in range(n):
        for p in params:
            p.grad = None
        s, c = ops.mlp_forward(spec, o, d, t, params, engine=_lib.ENGINES[os.environ.get("SPARF_OS_ENGINE", "tc_3x")])
        torch.autograd.backward([s, c], [gs, gc])
    torch.cuda.synchronize()


if __name__ == "__main__":
    main()
