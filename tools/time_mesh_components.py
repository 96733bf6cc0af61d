#!/usr/bin/env python
"""Time floater removal (ops.mesh_components, ops.mesh_select, mesh.keep_components) on the GPU, beside the marching
cubes that made the mesh and beside the host alternative.  Prints one JSON line per case and one with the device name
and power limit.

    python tools/time_mesh_components.py [--reps 5] [--cases dense256,dense512,sparse1024,sparse2048] [--no-host]

The field: a sphere of radius 0.6 at the origin plus small balls of radius 0.02 at the centres of a 0.2-spaced grid over
[-1.2, 1.2]^3 (those centres farther than 0.75 from the origin: 1520 balls, one component each), meshed at iso 0 by
ops.marching_cubes over the dense lattice (res 256, 512) or by ops.marching_cubes_sparse over its active blocks
(res 1024, 2048).  Per case, the best and median of --reps sync'd wall-clock times of:
  marching_cubes   the mesh's extraction from a field already on the device (dense: count + emit; sparse: count + emit);
  label            ops.mesh_components (its id check, the union-find, the face counts, and the read of C);
  select           ops.mesh_select keeping the sphere (its id and label checks, count + emit);
  keep_components  mesh.keep_components(largest=1), vertices gathered;
  host_copy, host_scipy  the host alternative: faces to the host, then scipy.sparse.csgraph.connected_components over
                   the vertex graph (edges (f0, f1), (f0, f2)) -- once, after one warm-up on a small graph.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np
import torch

from sparf_b200 import mesh, ops
from time_density import power_limit

RANGE = (-1.2, 1.2)
RADIUS, BALL, SPACING = 0.6, 0.02, 0.2


def field(p: torch.Tensor) -> torch.Tensor:
    """the sphere and the balls at points p [N, 3] (fp32): max of the signed distances, positive inside"""
    d = RADIUS - p.norm(dim=-1)
    n = round((RANGE[1] - RANGE[0]) / SPACING)
    cell = torch.floor((p - RANGE[0]) / SPACING).clamp_(0, n - 1)
    ctr = RANGE[0] + (cell + 0.5) * SPACING
    ball = torch.where(ctr.norm(dim=-1) > RADIUS + 0.15, BALL - (p - ctr).norm(dim=-1), torch.full_like(d, -1e9))
    return torch.maximum(d, ball)


def dense_volume(res):
    axis = mesh.lattice_axis(res, RANGE).cuda()
    n = axis.numel()
    vol = torch.empty(n, n, n, device="cuda")
    for i0, pts in mesh.lattice_slabs(axis, max(1, (1 << 22) // (n * n))):
        vol[i0:i0 + pts.shape[0] // (n * n)] = field(pts).view(-1, n, n)
    return vol


def sparse_blocks(res):
    axis = mesh.lattice_axis(res, RANGE).cuda()
    c = axis[::mesh.BLOCK]
    coarse = field(torch.stack(torch.meshgrid(c, c, c, indexing="ij"), -1).reshape(-1, 3)).view(c.numel(), c.numel(), -1)
    slots, ids = ops.mcubes_sparse_classify(coarse, 0.0)
    P = mesh.BLOCK + 1
    sigma = torch.empty(ids.numel(), P, P, P, device="cuda")
    per = 1 << 14
    for b0 in range(0, ids.numel(), per):
        nb = min(per, ids.numel() - b0)
        sigma[b0:b0 + nb] = field(ops.mcubes_sparse_points(axis, ids, b0, nb)).view(nb, P, P, P)
    return sigma, slots, ids


def timed(fn, reps):
    out, ts = None, []
    for _ in range(reps):
        torch.cuda.synchronize()
        t = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t) * 1e3)
    return out, dict(best_ms=round(min(ts), 3), median_ms=round(float(np.median(ts)), 3))


def host_components(faces_np, n_verts):
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    rows = np.concatenate([faces_np[:, 0], faces_np[:, 0]])
    cols = np.concatenate([faces_np[:, 1], faces_np[:, 2]])
    g = coo_matrix((np.ones(len(rows), np.int8), (rows, cols)), shape=(n_verts, n_verts))
    return connected_components(g, directed=False)[0]


def run_case(name, reps, host):
    kind = "dense" if name.startswith("dense") else "sparse"
    res = int(name[len(kind):])
    if kind == "dense":
        vol = dense_volume(res)
        mc = lambda: ops.marching_cubes(vol, 0.0)
    else:
        sigma, slots, ids = sparse_blocks(res)
        mc = lambda: ops.marching_cubes_sparse(sigma, res, slots, ids, 0.0)
    mc()                                                                        # warm-up
    (verts, faces), t_mc = timed(mc, reps)
    V, F = verts.shape[0], faces.shape[0]
    ops.mesh_components(faces, V)
    (labels, counts), t_label = timed(lambda: ops.mesh_components(faces, V), reps)
    keep = torch.zeros(counts.numel(), dtype=torch.uint8, device="cuda")
    keep[torch.argmax(counts)] = 1
    ops.mesh_select(faces, V, labels, keep)
    (vert_ids, kept_faces), t_select = timed(lambda: ops.mesh_select(faces, V, labels, keep), reps)
    m = dict(vertices=verts, faces=faces)
    mesh.keep_components(m, largest=1)
    _, t_keep = timed(lambda: mesh.keep_components(m, largest=1), reps)
    out = dict(case=name, res=res, V=V, F=F, components=counts.numel(), kept_V=vert_ids.numel(),
               kept_F=kept_faces.shape[0], marching_cubes=t_mc, label=t_label, select=t_select, keep_components=t_keep)
    if kind == "sparse":
        out["active_blocks"] = ids.numel()
    if host:
        host_components(np.array([[0, 1, 2]], np.int64), 3)
        torch.cuda.synchronize()
        t = time.perf_counter()
        f_np = faces.cpu().numpy()
        out["host_copy_ms"] = round((time.perf_counter() - t) * 1e3, 3)
        t = time.perf_counter()
        n = host_components(f_np, V)
        out["host_scipy_ms"] = round((time.perf_counter() - t) * 1e3, 3)
        assert n == counts.numel(), (n, counts.numel())
    print(json.dumps(out), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--cases", default="dense256,dense512,sparse1024,sparse2048")
    ap.add_argument("--no-host", action="store_true", help="skip the host path")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "time_mesh_components.py runs on a GPU"
    print(json.dumps(dict(device=torch.cuda.get_device_name(), power_limit_w=power_limit())), flush=True)
    for name in args.cases.split(","):
        run_case(name, args.reps, not args.no_host)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
