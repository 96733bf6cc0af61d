#!/usr/bin/env python
"""Time normal maps (Graph.set_normals) and mesh normals (ops.density_gradient) on the GPU.  Prints one JSON line with
the device name and power limit.

    python tools/time_normals.py [--engine tc_3x] [--reps 5]

(a) Full-image val renders of the octahedron scene of tools/time_occupancy.py (radius 0.6): 3 views of 300 x 400
    pixels, 128 coarse + 128 fine samples, through Graph.render_by_slices, dense, with res-128 occupancy grids, and with
    early termination (eps 1e-4, window 32).  Normals off and on alternate, best of --reps each; also the fraction of
    the samples (coarse + fine) with w != 0, the ones the normals differentiate.
(b) mesh.density_normals through the density backward (the autograd path it had before ops.density_gradient, copied
    below) against the new entry, at the vertex count of a res-512 sparse mesh of the same scene; the two outputs must
    be equal.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "golden"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch

import common
from sparf_b200 import mesh, occupancy, ops
from time_density import power_limit
from time_occupancy import octahedron_graph, sync_ms


@torch.no_grad()
def density_normals_backward(nerf, points, engine=None):
    """mesh.density_normals as it was: the gradient through ops.density_forward's backward, weight gradients included"""
    spec, trunk = nerf._spec(), mesh._trunk(nerf)
    out = torch.empty_like(points)
    for c0 in range(0, points.shape[0], mesh.NORMAL_CHUNK):
        x = points[c0:c0 + mesh.NORMAL_CHUNK].detach().clone().requires_grad_(True)
        with torch.enable_grad():
            raw, _ = ops.density_forward(spec, x, trunk, progress=nerf.progress.detach(), engine=engine, features=False)
            (g,) = torch.autograd.grad(raw.sum(), x)
        norm = g.norm(dim=-1, keepdim=True)
        out[c0:c0 + mesh.NORMAL_CHUNK] = torch.where(norm > 0, -g / norm, torch.zeros_like(g))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--engine", default="tc_3x")
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "time_normals.py measures on a GPU"
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
        grids = [occupancy.build_grid(opt, m, res=128) for m in net.get_network_components()]
        total = B * H * W * (128 + 256)
        for name in ("dense", "grid128", "termination"):
            net.set_occupancy(*(grids if name == "grid128" else (None, None)))
            net.set_early_termination(*((1e-4, 32) if name == "termination" else (None,)))
            times = {False: [], True: []}
            for rep in range(args.reps + 1):
                for normals in (False, True):
                    net.set_normals(normals)
                    e0 = ops.EVALS["bwd"]
                    ms, _ = sync_ms(lambda: render(net))
                    if normals:
                        visible = ops.EVALS["bwd"] - e0                 # the samples with w != 0, differentiated
                    if rep:                                             # rep 0 warms up
                        times[normals].append(ms)
            off, on = min(times[False]), min(times[True])
            out[name] = dict(render_ms=off, render_normals_ms=on, ratio=round(on / off, 3),
                             visible_fraction=round(visible / total, 4),
                             render_ms_all=[round(m, 2) for m in times[False]],
                             render_normals_ms_all=[round(m, 2) for m in times[True]])
        net.set_occupancy(None, None)
        net.set_early_termination(None)

        m = mesh.extract_mesh_sparse(dict(trimesh=dict(res=512, range=(-1.2, 1.2), thres=10.0)), net.nerf)
        verts = m["vertices"]
        new = mesh.density_normals(net.nerf, verts)
        old = density_normals_backward(net.nerf, verts)
        assert torch.equal(new, old), "density_normals changed"
        t_old, t_new = [], []
        for _ in range(args.reps):
            t_old.append(sync_ms(lambda: density_normals_backward(net.nerf, verts))[0])
            t_new.append(sync_ms(lambda: mesh.density_normals(net.nerf, verts))[0])
        out["mesh_normals"] = dict(vertices=verts.shape[0], backward_ms=min(t_old), gradient_ms=min(t_new),
                                   ratio=round(min(t_new) / min(t_old), 3))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
