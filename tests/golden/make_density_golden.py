#!/usr/bin/env python
"""Fixture of the density queries (tests/test_density_cpu.py, tests/test_density.py): the reference's own
NeRF.compute_raw_density (frequency_nerf.py:149-170) at arbitrary points, and the gradients of a fixed linear probe of its
two outputs.

    python tests/golden/make_density_golden.py      (needs the reference, see oracle/ref_loader.py)

Per case (default architecture, common.det_weights): points [2,37,5,3] uniform in [-1.5, 1.5]^3; stored: raw [2,37,5],
feat [2,37,5,256], and the gradients of  sum(a * raw) + sum(b * feat)  w.r.t. the points (in full), every trunk bias
(in full) and every trunk weight (strided sub-sample + fp64 sum of squares, as make_golden.py).  The inputs are rebuilt
by case_inputs() below, which does not need the reference.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [HERE, os.path.dirname(os.path.dirname(HERE))]

import common  # noqa: E402

PATH = os.path.join(HERE, "density_raw.npz")
SHAPE = (2, 37, 5)
CASES = {
    "plain": dict(seed=21, barf_c2f=None, progress=None),
    "c2f": dict(seed=22, barf_c2f=(0.1, 0.5), progress=0.3),
}


def case_inputs(name):
    """-> (opt, state dict, points [2,37,5,3], a [2,37,5], b [2,37,5,256]), fp32 on the CPU."""
    c = CASES[name]
    opt = common.make_opt(barf_c2f=c["barf_c2f"])
    sd = common.det_weights(opt, c["seed"], progress=c["progress"])
    rng = np.random.default_rng(c["seed"] + 6000)
    pts = torch.from_numpy(rng.uniform(-1.5, 1.5, size=SHAPE + (3,)).astype(np.float32))
    a = torch.from_numpy(rng.normal(0, 1, size=SHAPE).astype(np.float32))
    b = torch.from_numpy(rng.normal(0, 1, size=SHAPE + (opt.arch.layers_feat[-1],)).astype(np.float32))
    return opt, sd, pts, a, b


def probe(raw, feat, a, b):
    return (raw * a).sum() + (feat * b).sum()


def main():
    from oracle import ref_loader
    fn = ref_loader.load("renderer").frequency_nerf
    out = {}
    for name in CASES:
        opt, sd, pts, a, b = case_inputs(name)
        net = fn.NeRF(opt)
        net.load_state_dict(sd)
        pts = pts.clone().requires_grad_(True)
        raw, feat = net.compute_raw_density(opt, pts, fn.FrequencyEmbedder(opt))
        probe(raw, feat, a, b).backward()
        out[name + "/raw"] = raw.detach().numpy()
        out[name + "/feat"] = feat.detach().numpy()
        out[name + "/grad_points"] = pts.grad.numpy()
        for pname, p in net.named_parameters():
            if not pname.startswith("mlp_feat."):
                continue
            g = p.grad.numpy()
            key = "%s/grad_%s" % (name, pname)
            if pname.endswith("bias"):
                out[key] = g
            else:
                out[key + ".sub"] = common.subsample(g)
                out[key + ".sumsq"] = np.float64((g.astype(np.float64) ** 2).sum())
    np.savez_compressed(PATH, **out)
    print("%s: %d arrays, %.1f KB" % (PATH, len(out), os.path.getsize(PATH) / 1024))


if __name__ == "__main__":
    main()
