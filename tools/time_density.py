#!/usr/bin/env python
"""Throughput of the density queries (NeRF.compute_raw_density, ops.density_forward) on a grid of points, the kind of
query a marching-cubes or occupancy pass makes, against NeRF.forward on the same points and the PyTorch trunk of
tests/density_oracle.py (fp32 and TF32) on the same GPU.  CUDA events around whole passes after a warm-up chunk;
prints one JSON line.

    python tools/time_density.py [--grid 256] [--chunk 1048576] [--engines tc_3x,simt_fp32]

Network: the default architecture with its own tf_init weights (torch seed 0).  Points: the grid^3 lattice over
[-1.5, 1.5]^3, evaluated in chunks.  The backward figure is one forward + the gradient of raw.sum() w.r.t. the points
(the normals) over one chunk.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "golden")):
    sys.path.insert(0, p)
import torch

import common
from density_oracle import raw_density
from sparf_b200 import _lib, ops
from sparf_b200.frequency_nerf import NeRF


def elapsed_ms(fn, warm):
    warm()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        return float(out.strip().splitlines()[0])
    except Exception:
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--grid", type=int, default=256)
    ap.add_argument("--chunk", type=int, default=1 << 20)
    ap.add_argument("--engines", default="tc_3x,simt_fp32")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "time_density.py measures on a GPU"
    opt = common.make_opt()
    torch.manual_seed(0)
    nerf = NeRF(opt).cuda()
    trunk = nerf.kernel_params()[:2 * len(nerf.mlp_feat)]
    spec = nerf._spec()
    ax = torch.linspace(-1.5, 1.5, args.grid, device="cuda")
    grid = torch.stack(torch.meshgrid(ax, ax, ax, indexing="ij"), dim=-1).reshape(-1, 3)
    N, C = grid.shape[0], args.chunk
    chunks = [grid[i:i + C] for i in range(0, N, C)]
    ray = torch.tensor([0.3, -0.5, 0.8], device="cuda").expand(1, C, 3).contiguous()

    def over_grid(f):
        return lambda: [f(x) for x in chunks]

    res = dict(device=torch.cuda.get_device_name(), power_limit_w=power_limit(), points=N, chunk=C)
    with torch.no_grad():
        for name in args.engines.split(","):
            eng = _lib.ENGINES[name]
            ops.set_engine(eng)
            crd = lambda x: nerf.compute_raw_density(opt, x, None)
            raw_only = lambda x: ops.density_forward(spec, x, trunk, progress=nerf.progress, engine=eng, features=False)
            fwd = lambda x: nerf.forward(opt, x.view(1, -1, 1, 3), ray[:, :x.shape[0]], None, None)
            r = {}
            for key, f in (("compute_raw_density", crd), ("density_forward_no_features", raw_only), ("nerf_forward", fwd)):
                r[key + "_pts_per_s"] = N / (elapsed_ms(over_grid(f), lambda: f(chunks[0])) / 1e3)

            def normals():
                x = chunks[0].clone().requires_grad_(True)
                with torch.enable_grad():
                    raw, _ = ops.density_forward(spec, x, trunk, progress=nerf.progress, engine=eng, features=False)
                    torch.autograd.grad(raw.sum(), x)
            r["fwd_bwd_points_grad_pts_per_s"] = chunks[0].shape[0] / (elapsed_ms(normals, normals) / 1e3)
            res[name] = r
        ops.set_engine("auto")
        p = {k: v.detach() for k, v in nerf.state_dict().items()}
        ref = lambda x: raw_density(p, x, L_3D=opt.arch.posenc.L_3D, skip=tuple(opt.arch.skip), barf_c2f=opt.barf_c2f)
        tf32 = torch.backends.cuda.matmul.allow_tf32
        for key, allow in (("torch_fp32", False), ("torch_tf32", True)):
            torch.backends.cuda.matmul.allow_tf32 = allow
            res[key + "_raw_density_pts_per_s"] = N / (elapsed_ms(over_grid(ref), lambda: ref(chunks[0])) / 1e3)
        torch.backends.cuda.matmul.allow_tf32 = tf32
    print(json.dumps(res))


if __name__ == "__main__":
    main()
