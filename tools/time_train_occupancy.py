#!/usr/bin/env python
"""Time training steps with occupancy grids (Graph.set_training_occupancy) against dense ones, both captured as one CUDA
graph (GraphedStep) and replayed.  Prints one JSON line with the device name and power limit.

    python tools/time_train_occupancy.py [--engine tc_3x] [--steps 30]

A c2-shaped step: 3 views x 341 rays, 128 coarse samples (row "coarse"), and 128 coarse + 128 fine samples (row
"fine"), stratified, metric depth [1.5, 4.5]; render -> photometric loss -> backward into the parameters' gradients.
The scene is the analytic octahedron of tools/time_occupancy.py (σ = softplus(c - k |x|_1), both networks), whose radius
sets the kept fraction.  Reported per row and configuration (dense; radius 0.3 / 0.6 / 1.0 with grids of res 128 at
thres 0.01; radius 0.6 with thres 0, every cell occupied: the grid path's fixed cost): step_ms (CUDA events around
--steps replays, the median of 3 such runs) and the kept fraction of the coarse and fine samples of one step.  Also
refresh_ms: one occupancy.refresh_ of a res-128 grid.
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "golden"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch

import common
from sparf_b200 import occupancy, ops
from sparf_b200.graphs import GraphedStep
from time_density import power_limit
from time_occupancy import octahedron_graph, sync_ms

B, N = 3, 341


def kept_fraction(net, opt, pose, intr, H, W, ray_idx, depth_range, grids):
    """K / samples of one training render's coarse and fine passes, by the compaction the grid path runs"""
    with torch.no_grad():
        out = net.render(opt, pose, H=H, W=W, intr=intr, ray_idx=ray_idx, depth_range=depth_range, iter=None, mode="train")
    o, d = out["origins"].reshape(-1, 3), out["viewdirs"].reshape(-1, 3)
    fr = []
    for suffix, g in zip(("", "_fine"), grids):
        if "t" + suffix not in out:
            continue
        t = out["t" + suffix].reshape(o.shape[0], -1)
        fr.append(ops.occupancy_compact(g.bits, g.res, g.range, o, d, t)[0].numel() / t.numel())
    return fr


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--engine", default="tc_3x")
    ap.add_argument("--steps", type=int, default=30)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "time_train_occupancy.py measures on a GPU"
    ops.set_engine(args.engine)
    out = dict(device=torch.cuda.get_device_name(), power_limit_w=power_limit(), engine=args.engine, rays=B * N)
    Wimg = 400
    data = common.make_scene(3, B, 300, Wimg, focal=800.0)
    pose, intr = data.pose.cuda(), data.intr.cuda()
    depth_range = torch.tensor([1.5, 4.5], device="cuda")
    target = torch.rand(B, N, 3, device="cuda")
    ray_idx = torch.randperm(300 * Wimg, device="cuda")[:N]

    for row, fine in (("coarse", False), ("fine", True)):
        opt = common.make_opt(S=128, S_fine=128, fine=fine, stratified=True, depth_range=(1.5, 4.5))
        res_row = {}
        for name, radius, thres in (("dense", 0.6, None), ("r0.3", 0.3, 0.01), ("r0.6", 0.6, 0.01), ("r1.0", 1.0, 0.01),
                                    ("r0.6_all_occupied", 0.6, 0.0)):
            net = octahedron_graph(opt, radius)
            net.device_side_rng = True
            comps = net.get_network_components()
            params = [p for m in comps for p in m.parameters()]
            grids = [occupancy.build_grid(opt, m, res=128, thres=thres) for m in comps] if thres is not None else []
            net.set_training_occupancy(*(grids or [None]))

            def step():
                for p in params:
                    if p.grad is not None:
                        p.grad.zero_()
                o = net.render(opt, pose, H=300, W=Wimg, intr=intr, ray_idx=ray_idx, depth_range=depth_range, iter=None,
                               mode="train")
                loss = ((o["rgb"] - target) ** 2).mean() + (((o["rgb_fine"] - target) ** 2).mean() if fine else 0)
                loss.backward()
                return loss.detach()

            for p in params:
                p.grad = torch.zeros_like(p)
            g = GraphedStep(step, (), warmup=2)
            runs = []
            for _ in range(3):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.steps):
                    g()
                e1.record()
                torch.cuda.synchronize()
                runs.append(e0.elapsed_time(e1) / args.steps)
            r = dict(radius=radius, thres=thres, step_ms=statistics.median(runs), step_ms_runs=[round(x, 3) for x in runs])
            if grids:
                r["kept_fraction"] = kept_fraction(net, opt, pose, intr, 300, Wimg, ray_idx, depth_range, grids)
            res_row[name] = r
            del g
        out[row] = res_row

    opt = common.make_opt(S=128, depth_range=(1.5, 4.5))
    net = octahedron_graph(opt, 0.6)
    grid = occupancy.build_grid(opt, net.nerf, res=128)
    occupancy.refresh_(grid, opt, net.nerf)
    out["refresh_ms_res128"] = min(sync_ms(lambda: occupancy.refresh_(grid, opt, net.nerf))[0] for _ in range(5))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
