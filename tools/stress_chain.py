#!/usr/bin/env python
"""Repeat the MLP training step with a cold L2 and check that every repetition reproduces the first one: forward outputs
bit-exactly, gradients to rounding of the atomics.  STRESS_ENGINE=tc_3x (default) | tc_1x | tc_3x_w1 | simt_fp32."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "golden")):
    sys.path.insert(0, p)
import torch

import common
from sparf_b200 import _lib, ops


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 200
    R, S = (int(sys.argv[2]), int(sys.argv[3])) if len(sys.argv) > 3 else (1023, 128)
    opt = common.make_opt(S=S)
    sd = common.det_weights(opt, 0)
    keys = sum([["mlp_feat.%d.weight" % i, "mlp_feat.%d.bias" % i] for i in range(8)], []) + \
        ["mlp_rgb.0.weight", "mlp_rgb.0.bias", "mlp_rgb.1.weight", "mlp_rgb.1.bias"]
    params = [sd[k].cuda().requires_grad_(True) for k in keys]
    o = (torch.randn(R, 3, device="cuda") * 0.3).requires_grad_(True)
    d = torch.nn.functional.normalize(torch.randn(R, 3, device="cuda"), dim=-1).requires_grad_(True)
    t = torch.sort(torch.rand(R, S, device="cuda") * 4 + 1.2, dim=1).values
    spec = ops.MLPSpec()
    engine = _lib.ENGINES[os.environ.get("STRESS_ENGINE", "tc_3x")]
    gs, gc = torch.randn(R, S, device="cuda"), torch.randn(R, S, 3, device="cuda")
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    ref = None
    worst = 0.0
    for it in range(n):
        flush.fill_(it & 255)
        for p in params + [o, d]:
            p.grad = None
        s, c = ops.mlp_forward(spec, o, d, t, params, engine=engine)
        torch.autograd.backward([s, c], [gs, gc])
        torch.cuda.synchronize()
        cur = [s.detach().clone(), c.detach().clone()] + [p.grad.clone() for p in params + [o, d]]
        if ref is None:
            ref = cur
            continue
        assert torch.equal(cur[0], ref[0]) and torch.equal(cur[1], ref[1]), "forward differs at repetition %d" % it
        for a, b in zip(cur[2:], ref[2:]):
            err = ((a - b).abs().max() / b.abs().max().clamp_min(1e-30)).item()
            worst = max(worst, err)
            assert err < 1e-4, "gradient differs at repetition %d: %g" % (it, err)
    print("stress ok: %d repetitions, worst gradient deviation %.2e" % (n, worst))


if __name__ == "__main__":
    main()
