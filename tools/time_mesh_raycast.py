#!/usr/bin/env python
"""Time the mesh ray cast (ops.raycast, mesh.cull) on the GPU.  Prints one JSON line with the device name and power
limit, then one per case.

    python tools/time_mesh_raycast.py [--reps 5] [--cases sphere224,sphere448,sphere864,torus300,torus600,torus1160]
                                      [--views 3] [--height 1200] [--width 1600] [--brute 2000]

Each case is the marching-cubes sphere or torus of tools/time_mesh_distance.py at the given lattice resolution (about
0.4 M, 1.5 M and 5.7 M faces; unit size, centred at 0.5).  The rays are the pixel-centre rays of --views DTU-sized
views (default 3 x 1200 x 1600 = 5.76 M rays) on a ring around the shape at 2.2 sizes from its centre, looking at a
point off the centre, so that both hits and misses occur.  Per case: the best and median of --reps synchronised
wall-clock times of the grid build, of ops.raycast of all rays at the default grid and at 1/2 and 1/4 of its cells per
axis (the results must be the same bytes, and are checked), of a full mesh.cull of the views; then a chunked torch
brute force (every ray against every triangle, fp32 Moller-Trumbore) over --brute rays, checked against the grid's
faces where both hit, extrapolated linearly to all rays.
"""
import argparse
import json
import math
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch

from time_mesh_distance import shape_mesh, timed


def ring_cameras(n, H, W, radius=2.2, center=(0.5, 0.5, 0.5), focal=1.2):
    """pose_w2c [n, 3, 4], intr [3, 3] (CUDA fp32): n cameras on a tilted ring of the given radius around center, each
    looking at a point 0.15 off the centre, focal length focal * W"""
    c = torch.tensor(center, dtype=torch.float64)
    poses = []
    for i in range(n):
        a = 2 * math.pi * i / n + 0.3
        eye = c + radius * torch.tensor([math.cos(a), math.sin(a), 0.35], dtype=torch.float64)
        at = c + torch.tensor([0.15, -0.1, 0.05], dtype=torch.float64)
        z = (at - eye) / (at - eye).norm()
        x = torch.linalg.cross(z, torch.tensor([0.0, 0.0, 1.0], dtype=torch.float64))
        x = x / x.norm()
        y = torch.linalg.cross(z, x)
        R = torch.stack([x, y, z])          # world -> camera rows
        poses.append(torch.cat([R, (-R @ eye)[:, None]], 1))
    K = torch.tensor([[focal * W, 0, W / 2], [0, focal * W, H / 2], [0, 0, 1]], dtype=torch.float64)
    return torch.stack(poses).float().cuda(), K.float().cuda()


def brute_force(v, f, o, d, chunk=8):
    """the nearest two-sided Moller-Trumbore hit over all triangles, fp32 torch, chunk rays at a time -> (t, face)"""
    a, b, c = (v[f[:, k]][None] for k in range(3))
    e1, e2 = b - a, c - a
    t_out = torch.empty(o.shape[0], device=o.device)
    f_out = torch.empty(o.shape[0], dtype=torch.int64, device=o.device)
    for i0 in range(0, o.shape[0], chunk):
        oo, dd = o[i0:i0 + chunk, None], d[i0:i0 + chunk, None]
        dd = dd.expand(dd.shape[0], e2.shape[1], 3)
        p = torch.linalg.cross(dd, e2.expand_as(dd))
        det = (e1 * p).sum(-1)
        s = oo - a
        u = (s * p).sum(-1) / det
        q = torch.linalg.cross(s, e1.expand_as(s))
        w = (dd * q).sum(-1) / det
        t = (e2 * q).sum(-1) / det
        ok = (det != 0) & (u >= 0) & (w >= 0) & (u + w <= 1) & (t >= 0)
        t = torch.where(ok, t, torch.full_like(t, float("inf")))
        best = t.min(1)
        t_out[i0:i0 + chunk] = best.values
        f_out[i0:i0 + chunk] = torch.where(torch.isinf(best.values), -1, best.indices)
    return t_out, f_out


def run_case(name, reps, views, H, W, n_brute):
    from sparf_b200 import camera, mesh, ops
    kind = "sphere" if name.startswith("sphere") else "torus"
    res = int(name[len(kind):])
    v, f = shape_mesh(kind, res)
    pose, K = ring_cameras(views, H, W)
    o, d = camera.get_center_and_ray(pose, H, W, K.expand(views, 3, 3))
    o, d = o.reshape(-1, 3).contiguous(), d.reshape(-1, 3).contiguous()
    grid = ops.distance_grid(v, f)
    ops.raycast(grid, o, d)                                     # warm-up
    grid, t_grid = timed(lambda: ops.distance_grid(v, f), reps)
    (t, face, bary), t_cast = timed(lambda: ops.raycast(grid, o, d), reps)
    row = dict(case=name, V=v.shape[0], F=f.shape[0], rays=o.shape[0], hits=int((face >= 0).sum().item()),
               grid_dims=list(grid.dims), entries=grid.entries, grid=t_grid, raycast=t_cast)
    for div in (2, 4):
        dims = tuple(max(1, -(-n // div)) for n in grid.dims)
        g = ops.distance_grid(v, f, cells_per_axis=dims)
        ops.raycast(g, o, d)
        got, t_div = timed(lambda: ops.raycast(g, o, d), reps)
        same = all(torch.equal(a.view(torch.int32) if a.dtype == torch.float32 else a, b.view(torch.int32)
                               if b.dtype == torch.float32 else b) for a, b in zip(got, (t, face, bary)))
        row["raycast_1_%d" % div] = dict(t_div, grid_dims=list(g.dims), entries=g.entries, same_bytes=same)
        del g, got
    m = dict(vertices=v, faces=f)
    mesh.cull(m, pose, K, H, W)
    st = {}
    _, t_cull = timed(lambda: mesh.cull(m, pose, K, H, W, stats=st), reps)
    row.update(cull=t_cull, faces_after_cull=st["faces_after"])
    if n_brute:
        sel = torch.linspace(0, o.shape[0] - 1, n_brute, device="cuda").long()
        brute_force(v, f, o[sel[:16]], d[sel[:16]])
        (tb, fb), t_brute = timed(lambda: brute_force(v, f, o[sel], d[sel]), 1)
        both = (fb >= 0) & (face[sel] >= 0)
        row.update(brute_rays=n_brute, brute=t_brute,
                   brute_hit_agreement=float(((fb >= 0) == (face[sel] >= 0)).float().mean().item()),
                   brute_max_rel_t_diff=float(((tb - t[sel]).abs() / t[sel])[both].max().item()) if both.any() else 0.0,
                   brute_all_rays_s_extrapolated=round(t_brute["best_ms"] * o.shape[0] / n_brute / 1e3, 1))
    print(json.dumps(row), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--cases", default="sphere224,sphere448,sphere864,torus300,torus600,torus1160")
    ap.add_argument("--views", type=int, default=3)
    ap.add_argument("--height", type=int, default=1200)
    ap.add_argument("--width", type=int, default=1600)
    ap.add_argument("--brute", type=int, default=2000, help="rays of the torch brute force (0: skip)")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "time_mesh_raycast.py runs on a GPU"
    from time_density import power_limit
    print(json.dumps(dict(device=torch.cuda.get_device_name(), power_limit_w=power_limit())), flush=True)
    for name in args.cases.split(","):
        run_case(name, args.reps, args.views, args.height, args.width, args.brute)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
