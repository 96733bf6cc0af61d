#!/usr/bin/env python
"""Time training steps with early ray termination (Graph.set_training_termination), alone and on top of training
occupancy grids, against dense and grid-only steps, each captured as one CUDA graph (GraphedStep) and replayed.  Prints
one JSON line with the device name and power limit.

    python tools/time_train_termination.py [--engine tc_3x] [--steps 20] [--runs 3]

A c2-shaped step: 3 views x 341 rays, render -> photometric loss -> backward into the parameters' gradients.  Scenes:
  a_wall, a_octa_wall: the LLFF-shaped inverse-depth wall and octahedron-before-wall of tools/time_contraction.py,
      128 coarse samples, no fine pass, contracted grids (res 128, thres 0.01);
  b_sharp_octa: the octahedron of tools/time_occupancy.py with k 400, radius 1.0, 128 + 128 samples, box grids;
  c_soft_octa: k 40, radius 0.3 (nothing turns opaque), 128 + 128 samples, box grids, with eps = 0 as well.
Configurations are replayed in turn, --runs rounds of --steps replays each; step_ms is the median over the rounds.  Per
configuration: the kept fraction of each pass (samples with rgb != 0 in one no-gradient training render; for
termination also the oracle's count, tests/termination_oracle.py, from the same render's dense σ) and the max |Δ| of
rgb, depth and opacity against the same step without termination.
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

import numpy as np
import torch

import common
import termination_oracle as T
from sparf_b200 import occupancy, ops
from sparf_b200.graphs import GraphedStep
from time_contraction import CONTRACTION, forward_facing_poses
from time_contraction import scene_graph as contraction_scene
from time_density import power_limit
from time_occupancy import octahedron_graph

B, N = 3, 341


def _scene(name):
    """(net, opt, pose, intr, H, W, depth_range, grid kind)"""
    if name.startswith("a_"):
        H, W, focal = 378, 504, 407.0
        opt = common.make_opt(S=128, fine=False, stratified=True, depth_param="inverse", depth_range=(1, 0))
        net = contraction_scene(opt, "wall" if name == "a_wall" else "octa_wall")
        pose = forward_facing_poses().cuda()
        intr = torch.tensor([[focal, 0, W / 2.0], [0, focal, H / 2.0], [0, 0, 1]]).repeat(B, 1, 1).cuda()
        return net, opt, pose, intr, H, W, opt.nerf.depth.range, "contracted"
    k, radius = (400.0, 1.0) if name == "b_sharp_octa" else (40.0, 0.3)
    opt = common.make_opt(S=128, S_fine=128, fine=True, stratified=True, depth_range=(1.5, 4.5))
    net = octahedron_graph(opt, radius, k=k)
    data = common.make_scene(3, B, 300, 400, focal=800.0)
    return net, opt, data.pose.cuda(), data.intr.cuda(), 300, 400, torch.tensor([1.5, 4.5], device="cuda"), "box"


def _render(net, opt, pose, intr, H, W, ray_idx, depth_range, seed):
    torch.manual_seed(seed)
    return net.render(opt, pose, H=H, W=W, intr=intr, ray_idx=ray_idx, depth_range=depth_range, iter=None, mode="train")


@torch.no_grad()
def _oracle_kept(net, opt, out, grids, eps, window):
    """the oracle's kept fraction per pass from the dense σ of the same samples (grid lookup by the compaction)"""
    o, d = out["origins"].reshape(-1, 3), out["viewdirs"].reshape(-1, 3)
    fr = []
    for suffix, nerf, g in zip(("", "_fine"), net.get_network_components(), grids):
        if "t" + suffix not in out:
            continue
        t = out["t" + suffix].reshape(o.shape[0], -1)
        R, S = t.shape
        dense = nerf.forward_samples(opt, o.view(1, R, 3), d.view(1, R, 3), t.view(1, R, S, 1), mode="val")
        keep = None
        if g is not None:
            if g.contraction is None:
                idx = ops.occupancy_compact(g.bits, g.res, g.range, o, d, t)[0]
            else:
                idx = ops.contracted_compact(o, d, t, 0, S, None, g.bits, g.res, *g.contraction)[0]
            keep = np.zeros(R * S, bool)
            keep[idx.cpu().numpy()] = True
            keep = keep.reshape(R, S)
        ev = T.evaluated(dense["density_samples"].reshape(R, S).cpu().numpy(), t.cpu().numpy(), d.cpu().numpy(), eps,
                         window, keep)
        fr.append(round(float(ev.mean()), 4))
    return fr


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--engine", default="tc_3x")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--scenes", default="a_wall,a_octa_wall,b_sharp_octa,c_soft_octa")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "time_train_termination.py measures on a GPU"
    ops.set_engine(args.engine)
    out = dict(device=torch.cuda.get_device_name(), power_limit_w=power_limit(), engine=args.engine, rays=B * N)
    for name in args.scenes.split(","):
        net, opt, pose, intr, H, W, depth_range, kind = _scene(name)
        net.device_side_rng = True
        comps = net.get_network_components()
        params = [p for m in comps for p in m.parameters()]
        target = torch.rand(B, N, 3, device="cuda")
        ray_idx = torch.randperm(H * W, device="cuda")[:N]
        contraction = CONTRACTION if kind == "contracted" else None
        grids = [occupancy.build_grid(opt, m, res=128, thres=0.01, contraction=contraction) for m in comps]
        configs = [("dense", False, None), ("grid", True, None), ("term_w16", False, (1e-4, 16)), ("term_w32", False, (1e-4, 32)),
                   ("grid_term_w16", True, (1e-4, 16)), ("grid_term_w32", True, (1e-4, 32))]
        if name == "c_soft_octa":
            configs += [("grid_term_eps0_w16", True, (0.0, 16))]

        def setup(use_grid, term):
            net.set_training_occupancy(*(grids if use_grid else [None]))
            net.set_training_termination(*(term or (None,)))

        steps, res = {}, {}
        for cname, use_grid, term in configs:
            setup(use_grid, term)
            fine = opt.nerf.fine_sampling

            def step():
                for p in params:
                    if p.grad is not None:
                        p.grad.zero_()
                o = net.render(opt, pose, H=H, W=W, intr=intr, ray_idx=ray_idx, depth_range=depth_range, iter=None,
                               mode="train")
                loss = ((o["rgb"] - target) ** 2).mean() + (((o["rgb_fine"] - target) ** 2).mean() if fine else 0)
                loss.backward()
                return loss.detach()

            for p in params:
                p.grad = torch.zeros_like(p)
            steps[cname] = GraphedStep(step, (), warmup=2)
        times = {c: [] for c, _, _ in configs}
        for _ in range(args.runs):                        # configurations alternated within each round
            for cname, _, _ in configs:
                g = steps[cname]
                g()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.steps):
                    g()
                e1.record()
                torch.cuda.synchronize()
                times[cname].append(e0.elapsed_time(e1) / args.steps)
        renders = {}
        with torch.no_grad():
            for cname, use_grid, term in configs:
                setup(use_grid, term)
                renders[cname] = _render(net, opt, pose, intr, H, W, ray_idx, depth_range, 1)
        dense_ms = statistics.median(times["dense"])
        for cname, use_grid, term in configs:
            r = dict(step_ms=round(statistics.median(times[cname]), 3), step_ms_runs=[round(x, 3) for x in times[cname]])
            r["vs_dense"] = round(r["step_ms"] / dense_ms, 3)
            ren = renders[cname]
            r["kept_fraction"] = [round((ren["rgb_samples" + s].abs().sum(-1) != 0).float().mean().item(), 4)
                                  for s in ("", "_fine") if "rgb_samples" + s in ren]
            if term:
                setup(use_grid, None)
                r["oracle_kept_fraction"] = _oracle_kept(net, opt, ren, grids if use_grid else [None, None], *term)
                base = renders["grid" if use_grid else "dense"]
                for key in ("rgb", "depth", "opacity"):
                    for s in ("", "_fine"):
                        if key + s in ren:
                            r["max_abs_diff_" + key + s] = float("%.3g" % (ren[key + s] - base[key + s]).abs().max().item())
            res[cname] = r
        setup(False, None)
        out[name] = res
        del steps, renders
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
