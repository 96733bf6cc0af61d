#!/usr/bin/env python
"""Time the on-device occupancy grid update (occupancy.update_) against the full rebuild (occupancy.refresh_).  Prints
one JSON line with the device name and power limit.

    python tools/time_grid_update.py [--engine tc_3x] [--steps 160] [--every 16]

(a) calls: update_ of a res-128 grid with N = 2^16, 2^18, 2^20 samples (half uniform, half occupied), CUDA events around
    20 eager calls after a warm-up, the median of 3 such runs; refresh_ of a res-64 and a res-128 grid, a host clock
    around a synchronised call, the best of 5.
(b) training: the c2-shaped step of tools/time_train_occupancy.py (3 views x 341 rays, 128 coarse + 128 fine samples,
    stratified, metric depth [1.5, 4.5], the octahedron scene of radius 0.6) with res-128 grids at thres 0.01 on both
    networks, plus a fused Adam step, captured as one CUDA graph.  Every --every steps the grids are either rebuilt
    between replays (refresh_) or updated by a second captured graph (update_ with 4096 + 4096 samples per network,
    decay 0.95).  Reported: the amortised ms per step over --steps steps (host clock, synchronised at the ends) and the
    kept fraction of the coarse and fine samples of one step at the end.
"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "golden"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch

import common
from sparf_b200 import occupancy, ops
from sparf_b200.graphs import GraphedStep
from sparf_b200.optim import FlatParameters, FusedAdam
from time_density import power_limit
from time_occupancy import octahedron_graph, sync_ms
from time_train_occupancy import kept_fraction

B, N = 3, 341


def time_calls(fn, calls=20, runs=3):
    fn()
    out = []
    for _ in range(runs):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(calls):
            fn()
        e1.record()
        torch.cuda.synchronize()
        out.append(e0.elapsed_time(e1) / calls)
    return statistics.median(out)


def train(mode, args, pose, intr, depth_range, target, ray_idx):
    opt = common.make_opt(S=128, S_fine=128, fine=True, stratified=True, depth_range=(1.5, 4.5))
    net = octahedron_graph(opt, 0.6)
    net.device_side_rng = True
    comps = net.get_network_components()
    grids = [occupancy.build_grid(opt, m, res=128, thres=0.01, ema=mode == "update") for m in comps]
    net.set_training_occupancy(*grids)
    flat = FlatParameters(comps)
    adam = FusedAdam(flat, lr=1e-3)

    def step():
        flat.zero_grad()
        o = net.render(opt, pose, H=300, W=400, intr=intr, ray_idx=ray_idx, depth_range=depth_range, iter=None,
                       mode="train")
        loss = ((o["rgb"] - target) ** 2).mean() + ((o["rgb_fine"] - target) ** 2).mean()
        loss.backward()
        adam.step()
        return loss.detach()

    def update():
        for g, m in zip(grids, comps):
            occupancy.update_(g, m, 4096, 4096)

    g_step = GraphedStep(step, (), warmup=2)
    g_grid = GraphedStep(update, (), warmup=1) if mode == "update" else None
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for it in range(args.steps):
        if it % args.every == 0 and it > 0:
            if g_grid is not None:
                g_grid()
            else:
                for g, m in zip(grids, comps):
                    occupancy.refresh_(g, opt, m)
        g_step()
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) * 1e3 / args.steps
    return dict(step_ms=round(ms, 3), kept_fraction=[round(x, 4) for x in
                                                     kept_fraction(net, opt, pose, intr, 300, 400, ray_idx, depth_range,
                                                                   grids)],
                occupied_fraction=[round(g.occupied_fraction(), 4) for g in grids])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--engine", default="tc_3x")
    ap.add_argument("--steps", type=int, default=160)
    ap.add_argument("--every", type=int, default=16)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "time_grid_update.py measures on a GPU"
    ops.set_engine(args.engine)
    out = dict(device=torch.cuda.get_device_name(), power_limit_w=power_limit(), engine=args.engine)

    opt = common.make_opt(S=128, depth_range=(1.5, 4.5))
    net = octahedron_graph(opt, 0.6)
    calls = {}
    for res in (64, 128):
        grid = occupancy.build_grid(opt, net.nerf, res=res, thres=0.01, ema=True)
        occupancy.refresh_(grid, opt, net.nerf)
        calls["refresh_ms_res%d" % res] = round(min(sync_ms(lambda: occupancy.refresh_(grid, opt, net.nerf))[0]
                                                    for _ in range(5)), 3)
    grid = occupancy.build_grid(opt, net.nerf, res=128, thres=0.01, ema=True)
    for n in (2 ** 16, 2 ** 18, 2 ** 20):
        calls["update_ms_res128_n%d" % n] = round(time_calls(lambda: occupancy.update_(grid, net.nerf, n // 2, n // 2)), 4)
    out["calls"] = calls

    data = common.make_scene(3, B, 300, 400, focal=800.0)
    pose, intr = data.pose.cuda(), data.intr.cuda()
    depth_range = torch.tensor([1.5, 4.5], device="cuda")
    torch.manual_seed(0)
    target = torch.rand(B, N, 3, device="cuda")
    ray_idx = torch.randperm(300 * 400, device="cuda")[:N]
    out["training"] = dict(steps=args.steps, every=args.every)
    for mode in ("refresh", "update", "refresh", "update"):       # alternated: the second pair shows the spread
        out["training"].setdefault(mode, []).append(train(mode, args, pose, intr, depth_range, target, ray_idx))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
