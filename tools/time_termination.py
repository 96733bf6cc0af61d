#!/usr/bin/env python
"""Time early ray termination (sparf_b200.termination), alone and on top of occupancy grids, on the GPU.  Prints one
JSON line with the device name and power limit.

    python tools/time_termination.py [--engine tc_3x] [--reps 3] [--quick]

Workload: the val render of tools/time_occupancy.py, 3 views of 300 x 400 pixels (focal 800) from 3 units away through
Graph.render_by_slices.  Scenes (σ analytic, in both networks, 8 x 256 trunk):
  * octahedra σ = softplus(k (radius - |x|_1)), k 40, radius 0.3 / 0.6 / 1.0, and a sharp one (k 400, radius 1.0):
    metric depth [1.5, 4.5], 128 + 128 samples;
  * a wall σ = softplus(k (c - n.x)), k 400, n towards the cameras (every ray ends on it), c 0 (through the origin) and
    0.5 (closer to the cameras): metric depth [1.5, 4.5], 128 + 128 samples;
  * the same wall through the origin with inverse depth [1, 0], 128 samples, no fine network (the c4-like setting).
Configurations per scene: dense; grid only (res 128, thres 0.01; octahedra only); termination only and grid +
termination at eps in {1e-4, 1e-3} and window in {16, 32, 64}; termination at eps = 0 (nothing terminates: the path's
fixed cost).  Reported per configuration: render_ms (host clock around a synchronised render, best of --reps), the kept
fraction of the MLP sample evaluations (ops.EVALS, coarse + fine), the max |difference| of rgb / depth / opacity from
the dense render, coarse and fine, and the windows per pass.  Per-window fixed cost (phases_ms): one slice's coarse
pass (131 070 rays x 128 samples) at window 32, CUDA events around each phase: the compaction (count, the copy of K,
emit), the scatter (two index_copy_), the update, and the zero-fill of the outputs.  --quick: one scene, one config.
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
from sparf_b200 import occupancy, ops, termination
from sparf_b200.renderer import Graph
from time_density import power_limit
from time_occupancy import octahedron_weights, sync_ms


def wall_weights(opt, normal, c, k, seed=0):
    """state_dict of a NeRF whose density is softplus(k (c - n.x)): octahedron_weights' six units relu(+-x_a) carry
    any linear density row, here -k n.x + k c"""
    sd = octahedron_weights(opt, c=k * c, k=k, seed=seed)
    n_trunk = len(opt.arch.layers_feat) - 1
    name = common.layer_shapes(opt)[n_trunk - 1][0]
    w = sd[name + ".weight"]
    for a in range(3):
        w[0, 2 * a], w[0, 2 * a + 1] = -k * float(normal[a]), k * float(normal[a])
    return sd


def camera_normal(pose_w2c):
    """the unit mean direction of the camera centres (-R^T t): a wall across it faces every camera"""
    R, t = pose_w2c[:, :, :3].double().cpu(), pose_w2c[:, :, 3].double().cpu()
    centres = -(R.transpose(1, 2) @ t[..., None])[..., 0]
    n = centres.mean(0)
    n = n / n.norm()
    assert (centres @ n).min() > 1.0, "the cameras do not all face one side of the wall"
    return n.numpy()


def scene_graph(opt, scene, normal=None):
    """Graph with both networks holding the scene: ("octa", radius, k) or ("wall", c, k)"""
    net = Graph(opt, torch.device("cuda"))
    kind, a, k = scene
    for i, m in enumerate(net.get_network_components()):
        sd = octahedron_weights(opt, c=k * a, k=k, seed=i) if kind == "octa" else wall_weights(opt, normal, a, k, seed=i)
        m.load_state_dict(sd)
    return net


def phase_times(net, opt, pose, intr, W, n_rays, window=32, eps=1e-4, reps=5):
    """CUDA-event times of the phases of termination.forward_samples on one slice's coarse pass, summed over its
    windows (best of reps)"""
    B = pose.shape[0]
    center, ray = ops.raygen(pose, intr, W, ray_idx=torch.arange(n_rays // B, device="cuda"))
    R = center.shape[0] * center.shape[1]
    o, d = center.reshape(R, 3), ray.reshape(R, 3)
    S = opt.nerf.sample_intvs
    t = ops.sample_depth(R, S, 1.5, 3.0, device="cuda")
    nerf = net.nerf
    limit = termination.tau_max(eps)
    best = None
    for _ in range(reps + 1):
        ev = {}

        def mark(name):
            e = torch.cuda.Event(enable_timing=True)
            e.record()
            ev.setdefault(name, []).append(e)

        mark("zero0")
        sigma = torch.zeros(R, S, device="cuda")
        rgb = torch.zeros(R * S, 3, device="cuda")
        alive = torch.ones(R, dtype=torch.uint8, device="cuda")
        tau = torch.zeros(R, device="cuda")
        mark("zero1")
        for k0 in range(0, S, window):
            k1 = min(k0 + window, S)
            mark("compact0")
            idx, o_k, d_k, t_k = ops.termination_compact(o, d, t, k0, k1, alive)
            mark("compact1")
            if idx.numel():
                s_k, r_k = ops.mlp_forward(nerf._spec(), o_k, d_k, t_k, nerf.kernel_params(), progress=nerf.progress)
                mark("scatter0")
                sigma.view(-1).index_copy_(0, idx, s_k.view(-1))
                rgb.index_copy_(0, idx, r_k.view(-1, 3))
                mark("scatter1")
            if k1 < S:
                mark("update0")
                ops.termination_update(sigma, t, d, k0, k1, limit, tau, alive)
                mark("update1")
        torch.cuda.synchronize()
        ms = {p: sum(a.elapsed_time(b) for a, b in zip(ev[p + "0"], ev[p + "1"])) for p in
              ("zero", "compact", "scatter", "update")}
        ms["windows"] = len(ev["compact0"])
        if best is None or sum(v for k, v in ms.items() if k != "windows") < sum(v for k, v in best.items() if k != "windows"):
            best = ms
    best["rays"] = R
    return best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--engine", default="tc_3x")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--quick", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "time_termination.py measures on a GPU"
    ops.set_engine(args.engine)
    out = dict(device=torch.cuda.get_device_name(), power_limit_w=power_limit(), engine=args.engine)
    B, H, W = 3, 300, 400
    data = common.make_scene(3, B, H, W, focal=800.0)
    pose, intr = data.pose.cuda(), data.intr.cuda()
    normal = camera_normal(data.pose)
    metric = common.make_opt(S=128, S_fine=128, fine=True, depth_range=(1.5, 4.5))
    inverse = common.make_opt(S=128, fine=False, depth_param="inverse", depth_range=(1, 0))
    scenes = [("octa_r0.3_k40", metric, ("octa", 0.3, 40.0)), ("octa_r0.6_k40", metric, ("octa", 0.6, 40.0)),
              ("octa_r1.0_k40", metric, ("octa", 1.0, 40.0)), ("octa_r1.0_k400", metric, ("octa", 1.0, 400.0)),
              ("wall_c0_k400", metric, ("wall", 0.0, 400.0)), ("wall_c0.5_k400", metric, ("wall", 0.5, 400.0)),
              ("wall_c0_k400_inverse", inverse, ("wall", 0.0, 400.0))]
    term = [(eps, w) for eps in (1e-4, 1e-3) for w in (16, 32, 64)]
    if args.quick:
        scenes, term = scenes[3:4], [(1e-4, 32)]

    with torch.no_grad():
        for name, opt, scene in scenes:
            net = scene_graph(opt, scene, normal)
            depth_range = opt.nerf.depth.range if opt.nerf.depth.param == "inverse" else torch.tensor([1.5, 4.5], device="cuda")
            render = lambda: net.render_by_slices(opt, pose, H, W, intr, depth_range, iter=None, mode="val")
            fine = opt.nerf.fine_sampling
            dense_evals = B * H * W * (opt.nerf.sample_intvs + (opt.nerf.sample_intvs + opt.nerf.sample_intvs_fine
                                                                if fine else 0))
            grids = [occupancy.build_grid(opt, m, res=128, thres=0.01) for m in net.get_network_components()] \
                if scene[0] == "octa" else None
            configs = [("dense", None, None)] + ([("grid", grids, None)] if grids else [])
            configs += [("term_eps%g_w%d" % tw, None, tw) for tw in term] + [("term_eps0_w32", None, (0.0, 32))]
            if grids:
                configs += [("grid_term_eps%g_w%d" % tw, grids, tw) for tw in term]
            res, dense = {}, None
            for cname, g, tw in configs:
                net.set_occupancy(*(g or (None, None)))
                net.set_early_termination(*(tw or (None,)))
                render()                                                 # warm-up
                e0 = ops.EVALS["fwd"]
                ms = [sync_ms(render) for _ in range(args.reps)]
                ret = ms[-1][1]
                if dense is None:
                    dense = ret
                r = dict(render_ms=round(min(m for m, _ in ms), 2), render_ms_all=[round(m, 2) for m, _ in ms],
                         kept_fraction=round((ops.EVALS["fwd"] - e0) / args.reps / dense_evals, 4))
                if tw is not None:
                    r["windows_per_pass"] = [-(-opt.nerf.sample_intvs // tw[1])] + \
                        ([-(-(opt.nerf.sample_intvs + opt.nerf.sample_intvs_fine) // tw[1])] if fine else [])
                for key in ("rgb", "depth", "opacity") + (("rgb_fine", "depth_fine", "opacity_fine") if fine else ()):
                    r["max_abs_diff_" + key] = float("%.3g" % (ret[key] - dense[key]).abs().max().item())
                r["opaque_fraction"] = round((dense["opacity_fine" if fine else "opacity"] > 0.9999).float().mean().item(), 4)
                res[cname] = r
            net.set_occupancy(None)
            net.set_early_termination(None)
            res["dense_vs_eps0_overhead"] = round(res["term_eps0_w32"]["render_ms"] / res["dense"]["render_ms"] - 1, 4)
            out[name] = res

        net = scene_graph(metric, ("wall", 0.0, 400.0), normal)
        out["phases_ms_wall_coarse_w32"] = phase_times(net, metric, pose, intr, W, net.full_image_rays_per_launch)
        out["phases_ms_wall_coarse_w16"] = phase_times(net, metric, pose, intr, W, net.full_image_rays_per_launch,
                                                       window=16)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
