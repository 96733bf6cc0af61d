#!/usr/bin/env python
"""Time contracted occupancy grids (sparf_b200.occupancy, contraction = (center, radius)) on the GPU, against the dense
render, early ray termination alone and the box grid.  Prints one JSON line with the device name and power limit.

    python tools/time_contraction.py [--engine tc_3x] [--reps 3]

Workload: a val render in LLFF's shape through Graph.render_by_slices: 3 forward-facing views of 378 x 504 pixels
(focal 407) from camera centres at x = -0.1, 0, 0.1 looking down +z, inverse depth [1, 0], 128 samples, no fine
network (8 x 256 trunk).  Scenes (σ analytic, tools/time_termination.py's constructions):
  * wall: σ = softplus(400 (z - 3)), every ray ends on it at depth 3;
  * octa_wall: an octahedron σ = softplus(40 (0.5 - |x - (0, 0, 2)|_1)) in front of that wall, σ the softplus of the
    max of the two.
Configurations, alternated rep by rep: dense; termination (eps 1e-4, window 16); the box grid of opt.trimesh
([-1.2, 1.2]^3, res 128); the contracted grid (center (0, 0, 0), radius 1.33, res 128); contracted grid +
termination.  All grids at thres 0.01.  Reported per configuration: render_ms (host clock around a synchronised render,
best of --reps), the kept fraction of the MLP sample evaluations (ops.EVALS), and the max |difference| of rgb / depth /
opacity from the dense render.  Also: the contracted grid's build time (build_grid) at res 128 and 256.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "golden"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np
import torch

import common
from sparf_b200 import occupancy, ops
from sparf_b200.renderer import Graph
from time_density import power_limit
from time_occupancy import octahedron_weights, sync_ms
from time_termination import wall_weights

CONTRACTION = ((0.0, 0.0, 0.0), 1.33)    # the camera centre and the LLFF loader's near bound


def octa_wall_weights(opt, center, radius, k_octa, wall_z, k_wall, seed=0):
    """state_dict of a NeRF whose density is softplus(max(a, b)), a = k_octa (radius - |x - center|_1) (an
    octahedron), b = k_wall (z - wall_z) (a wall facing -z): layer 0 makes relu(+-(x_a - center_a)), layer 1 adds a
    seventh unit relu(a - b), the next layers pass the seven units through, and the density row is b + relu(a - b)."""
    sd = octahedron_weights(opt, c=0.0, k=0.0, seed=seed)
    shapes = common.layer_shapes(opt)
    n_trunk = len(opt.arch.layers_feat) - 1
    cz_off = float(center[2]) - wall_z                       # z - wall_z = (u4 - u5) + cz_off
    for li, (name, k_out, k_in) in enumerate(shapes[:n_trunk]):
        w, b = sd[name + ".weight"], sd[name + ".bias"]
        if li == 0:
            for a in range(3):
                b[2 * a], b[2 * a + 1] = -float(center[a]), float(center[a])
        elif li < n_trunk - 1:
            w[6, 6] = 1.0
            if li == 1:
                w[6, 6] = 0.0
                w[6, :6] = -k_octa
                w[6, 4] -= k_wall
                w[6, 5] += k_wall
                b[6] = k_octa * radius - k_wall * cz_off
        else:
            w[0] = 0.0
            w[0, 4], w[0, 5], w[0, 6], b[0] = k_wall, -k_wall, 1.0, k_wall * cz_off
            w[7, 6] = 1.0
    return sd


def scene_graph(opt, kind):
    net = Graph(opt, torch.device("cuda"))
    if kind == "wall":
        sd = wall_weights(opt, (0.0, 0.0, -1.0), -3.0, 400.0)
    else:
        sd = octa_wall_weights(opt, (0.0, 0.0, 2.0), 0.5, 40.0, 3.0, 400.0)
    net.nerf.load_state_dict(sd)
    return net


def forward_facing_poses(xs=(-0.1, 0.0, 0.1)):
    """w2c [B,3,4]: identity rotation, camera centre (x, 0, 0)"""
    return torch.tensor([[[1, 0, 0, -x], [0, 1, 0, 0], [0, 0, 1, 0]] for x in xs], dtype=torch.float32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--engine", default="tc_3x")
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "time_contraction.py measures on a GPU"
    ops.set_engine(args.engine)
    out = dict(device=torch.cuda.get_device_name(), power_limit_w=power_limit(), engine=args.engine)
    B, H, W, focal = 3, 378, 504, 407.0
    pose = forward_facing_poses().cuda()
    intr = torch.tensor([[focal, 0, W / 2.0], [0, focal, H / 2.0], [0, 0, 1]]).repeat(B, 1, 1).cuda()
    opt = common.make_opt(S=128, fine=False, depth_param="inverse", depth_range=(1, 0))
    dense_evals = B * H * W * opt.nerf.sample_intvs

    with torch.no_grad():
        net = scene_graph(opt, "wall")
        for res in (128, 256):
            occupancy.build_grid(opt, net.nerf, res=res, contraction=CONTRACTION)
            ms = min(sync_ms(lambda: occupancy.build_grid(opt, net.nerf, res=res, contraction=CONTRACTION))[0]
                     for _ in range(3))
            out["contracted_build_res%d_ms" % res] = round(ms, 2)

        for kind in ("wall", "octa_wall"):
            net = scene_graph(opt, kind)
            render = lambda: net.render_by_slices(opt, pose, H, W, intr, opt.nerf.depth.range, iter=None, mode="val")
            box = occupancy.build_grid(opt, net.nerf, res=128, thres=0.01)
            con = occupancy.build_grid(opt, net.nerf, res=128, thres=0.01, contraction=CONTRACTION)
            configs = [("dense", None, None), ("termination", None, (1e-4, 16)), ("box_grid", box, None),
                       ("contracted_grid", con, None), ("contracted_grid_termination", con, (1e-4, 16))]
            ms = {name: [] for name, _, _ in configs}
            kept, rets = {}, {}
            for rep in range(args.reps + 1):                   # rep 0 warms up
                for name, g, tw in configs:
                    net.set_occupancy(g)
                    net.set_early_termination(*(tw or (None,)))
                    e0 = ops.EVALS["fwd"]
                    t_ms, ret = sync_ms(render)
                    if rep:
                        ms[name].append(t_ms)
                    kept[name] = (ops.EVALS["fwd"] - e0) / dense_evals
                    rets[name] = ret
            net.set_occupancy(None)
            net.set_early_termination(None)
            res = dict(box_occupied_fraction=round(box.occupied_fraction(), 4),
                       contracted_occupied_fraction=round(con.occupied_fraction(), 4),
                       dense_opacity_min=round(rets["dense"]["opacity"].min().item(), 6))
            for name, _, _ in configs:
                r = dict(render_ms=round(min(ms[name]), 2), render_ms_all=[round(m, 2) for m in ms[name]],
                         kept_fraction=round(kept[name], 4))
                r["vs_dense"] = round(r["render_ms"] / min(ms["dense"]), 3)
                for key in ("rgb", "depth", "opacity"):
                    r["max_abs_diff_" + key] = float("%.3g" % (rets[name][key] - rets["dense"][key]).abs().max().item())
                res[name] = r
            out[kind] = res
            del rets
    print(json.dumps(out))


if __name__ == "__main__":
    main()
