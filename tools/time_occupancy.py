#!/usr/bin/env python
"""Time empty-space skipping (sparf_b200.occupancy) on the GPU.  Prints one JSON line with the device name and power
limit.

    python tools/time_occupancy.py [--engine tc_3x] [--reps 5]

Scene: an analytic octahedron σ = softplus(c - k |x|_1), c = k * radius, k = 40 (octahedron_weights), in both the
coarse and the fine network (8 x 256 trunk, 128-wide colour head); 3 views of 300 x 400 pixels (focal 800) from 3 units away,
metric depth [1.5, 4.5], 128 coarse + 128 fine samples, a val render through Graph.render_by_slices.  The radius sets
the kept fraction.  Reported:
  * build_ms: occupancy.build_grid (density_grid + ops.occupancy_build) at res 128 and 256, and occupancy_build_ms
    alone;
  * per configuration (dense; radius 0.3 / 0.6 / 1.0 with thres 0.01 at res 128; radius 0.6 with thres 0, where every
    cell is occupied): render_ms (host clock around a synchronised render, best of --reps), the kept fraction of the
    MLP sample evaluations (coarse + fine), and the max |difference| of rgb / depth / opacity (fine and coarse) from the
    dense render;
  * compact_ms: one ops.occupancy_compact call (count, the copy of K, emit) on one slice's coarse and fine samples.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "golden"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np
import torch

import common
from sparf_b200 import mesh, occupancy, ops
from sparf_b200.renderer import Graph
from time_density import power_limit


def octahedron_weights(opt, c, k, seed=0):
    """state_dict of a NeRF whose density is softplus(c - k |x|_1): layer 0 maps the raw x channels to relu(+-x_a), the
    next layers pass those six units through (the skip layer's weights on the encoding are 0), the density row is
    c - k * their sum.  The features are the six units; the colour head has small random weights, so the colour depends
    on the position and the view direction."""
    rng = np.random.default_rng(seed)
    sd = {}
    n_trunk = len(opt.arch.layers_feat) - 1
    for li, (name, k_out, k_in) in enumerate(common.layer_shapes(opt)):
        w = np.zeros((k_out, k_in), np.float32)
        b = np.zeros(k_out, np.float32)
        if li == 0:
            for a in range(3):
                w[2 * a, a], w[2 * a + 1, a] = 1, -1
        elif li < n_trunk - 1:
            w[np.arange(6), np.arange(6)] = 1
        elif li == n_trunk - 1:
            w[0, :6], b[0] = -k, c
            w[1 + np.arange(6), np.arange(6)] = 1
        else:
            w = rng.normal(0, 0.3, (k_out, k_in)).astype(np.float32)
            b = rng.normal(0, 0.1, k_out).astype(np.float32)
        sd[name + ".weight"], sd[name + ".bias"] = torch.from_numpy(w), torch.from_numpy(b)
    sd["progress"] = torch.tensor(1.0)
    return sd


def octahedron_graph(opt, radius, k=40.0):
    net = Graph(opt, torch.device("cuda"))
    for i, m in enumerate(net.get_network_components()):
        m.load_state_dict(octahedron_weights(opt, c=k * radius, k=k, seed=i))
    return net


def sync_ms(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--engine", default="tc_3x")
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "time_occupancy.py measures on a GPU"
    ops.set_engine(args.engine)
    out = dict(device=torch.cuda.get_device_name(), power_limit_w=power_limit(), engine=args.engine)
    B, H, W = 3, 300, 400
    opt = common.make_opt(S=128, S_fine=128, fine=True, depth_range=(1.5, 4.5))
    data = common.make_scene(3, B, H, W, focal=800.0)
    pose, intr = data.pose.cuda(), data.intr.cuda()
    depth_range = torch.tensor([1.5, 4.5], device="cuda")
    render = lambda net: net.render_by_slices(opt, pose, H, W, intr, depth_range, iter=None, mode="val")

    with torch.no_grad():
        net = octahedron_graph(opt, 0.6)
        for res in (128, 256):
            occupancy.build_grid(opt, net.nerf, res=res)
            b_ms = min(sync_ms(lambda: occupancy.build_grid(opt, net.nerf, res=res))[0] for _ in range(3))
            sigma = mesh.density_grid(opt, net.nerf, res=res)
            ops.occupancy_build(sigma, 0.01)
            o_ms = min(sync_ms(lambda: ops.occupancy_build(sigma, 0.01))[0] for _ in range(3))
            out["build_res%d" % res] = dict(build_ms=b_ms, occupancy_build_ms=o_ms)
            del sigma

        configs = [("dense", 0.6, None), ("r0.3", 0.3, 0.01), ("r0.6", 0.6, 0.01), ("r1.0", 1.0, 0.01),
                   ("r0.6_thres0", 0.6, 0.0)]
        dense_evals = B * H * W * (128 + 256)
        dense = {}
        for name, radius, thres in configs:
            net = octahedron_graph(opt, radius)
            if radius not in dense:
                dense[radius] = render(net)
            grids = [occupancy.build_grid(opt, m, res=128, thres=thres) for m in net.get_network_components()] \
                if thres is not None else [None, None]
            net.set_occupancy(*grids)
            render(net)                                                 # warm-up
            e0 = ops.EVALS["fwd"]
            ms = [sync_ms(lambda: render(net)) for _ in range(args.reps)]
            ret = ms[-1][1]
            r = dict(radius=radius, thres=thres, render_ms=min(m for m, _ in ms),
                     render_ms_all=[round(m, 2) for m, _ in ms],
                     kept_fraction=(ops.EVALS["fwd"] - e0) / args.reps / dense_evals)
            for key in ("rgb", "depth", "opacity", "rgb_fine", "depth_fine", "opacity_fine"):
                r["max_abs_diff_" + key] = (ret[key] - dense[radius][key]).abs().max().item()
            if thres is not None:
                r["occupied_fraction"] = [g.occupied_fraction() for g in grids]
            out[name] = r

        # one slice's compaction (count, copy of K, emit), coarse and fine sample sets
        net = octahedron_graph(opt, 0.6)
        g = occupancy.build_grid(opt, net.nerf, res=128)
        n = net.full_image_rays_per_launch // B
        ray_idx = torch.arange(n, device="cuda")
        center, ray = ops.raygen(pose, intr, W, ray_idx=ray_idx)
        o, d = center.reshape(-1, 3), ray.reshape(-1, 3)
        for S in (128, 256):
            t = ops.sample_depth(o.shape[0], S, 1.5, 3.0, device="cuda")
            ops.occupancy_compact(g.bits, g.res, g.range, o, d, t)
            c_ms = min(sync_ms(lambda: ops.occupancy_compact(g.bits, g.res, g.range, o, d, t))[0] for _ in range(5))
            out["compact_S%d" % S] = dict(rays=o.shape[0], compact_ms=c_ms)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
