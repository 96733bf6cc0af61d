#!/usr/bin/env python
"""Time the closest-point queries of mesh.compare (ops.distance_grid, ops.closest_points) on the GPU.  Prints one JSON
line with the device name and power limit, then one per case.

    python tools/time_mesh_distance.py [--reps 5] [--cases sphere224,sphere448,sphere864,torus300,torus600,torus1160]
                                       [--queries 1000000] [--brute 10000]

Each case is a marching-cubes sphere or torus at the given lattice resolution (about 0.4 M, 1.6 M and 6 M faces), and
the queries are --queries surface samples of the same shape extracted at 3/4 of that resolution (another
tessellation of the surface).  Per case: the best and median of --reps synchronised wall-clock times of the grid build
(count, one read of the totals, fill) and of the query; then the same queries against a point cloud of --queries
samples of the mesh (a point grid); and a chunked torch brute force (every query against every triangle, fp32) over
--brute queries, checked against the grid's distances, extrapolated linearly to all queries.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch


def shape_volume(kind, res, device):
    """a signed field on a (res+1)^3 lattice whose zero set is a sphere (radius 0.45 res) or a torus (0.3 / 0.12 res)"""
    n = res + 1
    t = torch.arange(n, device=device, dtype=torch.float32) - (n - 1) / 2 - 0.13
    vol = torch.empty(n, n, n, device=device)
    for i in range(n):
        x, y, z = t[i], t[:, None], t[None, :]
        if kind == "sphere":
            vol[i] = 0.45 * res - torch.sqrt(x * x + y * y + z * z)
        else:
            q = torch.sqrt(x * x + y * y) - 0.3 * res
            vol[i] = 0.12 * res - torch.sqrt(q * q + z * z)
    return vol


def shape_mesh(kind, res, device="cuda"):
    """(vertices [V, 3] in units of the shape's size: index / res, faces [F, 3])"""
    from sparf_b200 import ops
    v, f = ops.marching_cubes(shape_volume(kind, res, device), 0.0)
    return v / res, f


def timed(fn, reps):
    out, ts = None, []
    for _ in range(reps):
        torch.cuda.synchronize()
        t = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t) * 1e3)
    ts.sort()
    return out, dict(best_ms=round(ts[0], 3), median_ms=round(ts[len(ts) // 2], 3))


def brute_force(v, f, p, chunk=16):
    """min over all triangles of the closest-point distance, fp32 torch, chunk queries at a time"""
    a, b, c = (v[f[:, k]] for k in range(3))
    out = torch.empty(p.shape[0], device=p.device)
    for i0 in range(0, p.shape[0], chunk):
        q = p[i0:i0 + chunk, None]
        out[i0:i0 + chunk] = torch_closest_d2(q, a[None], b[None], c[None]).min(1).values.sqrt()
    return out


def torch_closest_d2(p, a, b, c):
    """mesh_distance_oracle.closest_on_triangle's squared distance in torch"""
    def seg(u, w):
        d = w - u
        l = (d * d).sum(-1)
        t = torch.where(l > 0, ((p - u) * d).sum(-1) / l.clamp_min(1e-38), torch.zeros_like(l)).clamp(0, 1)
        r = p - (u + t[..., None] * d)
        return (r * r).sum(-1)
    d2 = torch.minimum(torch.minimum(seg(a, b), seg(b, c)), seg(c, a))
    ab, ac, ap = b - a, c - a, p - a
    n = torch.linalg.cross(ab.double(), ac.double()).float().expand_as(ap)
    nn = (n * n).sum(-1)
    dot = lambda x, y: (x * y).sum(-1)
    inside = ((nn > 0) & (dot(n, torch.linalg.cross(ab.expand_as(ap), ap)) >= 0)
              & (dot(n, torch.linalg.cross((c - b).expand_as(ap), p - b)) >= 0)
              & (dot(n, torch.linalg.cross((a - c).expand_as(ap), p - c)) >= 0))
    df = dot(n, ap) ** 2 / nn.clamp_min(1e-38)
    return torch.where(inside, torch.minimum(df, d2), d2)


def run_case(name, reps, n_queries, n_brute):
    from sparf_b200 import mesh, ops
    kind = "sphere" if name.startswith("sphere") else "torus"
    res = int(name[len(kind):])
    v, f = shape_mesh(kind, res)
    qv, qf = shape_mesh(kind, res * 3 // 4)
    pts = mesh.sample_surface(dict(vertices=qv, faces=qf), n_queries, seed=1)
    del qv, qf
    ops.closest_points(ops.distance_grid(v, f), pts)           # warm-up
    grid, t_grid = timed(lambda: ops.distance_grid(v, f), reps)
    (d, _, _), t_query = timed(lambda: ops.closest_points(grid, pts), reps)
    cloud = mesh.sample_surface(dict(vertices=v, faces=f), n_queries, seed=2)
    ops.closest_points(ops.distance_grid(cloud), pts)
    pgrid, t_pgrid = timed(lambda: ops.distance_grid(cloud), reps)
    _, t_pquery = timed(lambda: ops.closest_points(pgrid, pts), reps)
    row = dict(case=name, V=v.shape[0], F=f.shape[0], queries=pts.shape[0], grid_dims=list(grid.dims),
               entries=grid.entries, grid=t_grid, query=t_query, mean_dist=round(d.double().mean().item(), 7),
               cloud_points=cloud.shape[0], cloud_grid_dims=list(pgrid.dims), cloud_grid=t_pgrid, cloud_query=t_pquery)
    if n_brute:
        sub = pts[:n_brute]
        brute_force(v, f, sub[:64])
        db, t_brute = timed(lambda: brute_force(v, f, sub), 1)
        err = (db - d[:n_brute]).abs().max().item()
        row.update(brute_queries=n_brute, brute=t_brute, brute_max_abs_diff=err,
                   brute_all_queries_s_extrapolated=round(t_brute["best_ms"] * pts.shape[0] / n_brute / 1e3, 1))
    print(json.dumps(row), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--cases", default="sphere224,sphere448,sphere864,torus300,torus600,torus1160")
    ap.add_argument("--queries", type=int, default=1_000_000)
    ap.add_argument("--brute", type=int, default=10_000, help="queries of the torch brute force (0: skip)")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "time_mesh_distance.py runs on a GPU"
    from time_density import power_limit
    print(json.dumps(dict(device=torch.cuda.get_device_name(), power_limit_w=power_limit())), flush=True)
    for name in args.cases.split(","):
        run_case(name, args.reps, args.queries, args.brute)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
