#!/usr/bin/env python
"""Time the mesh simplification (ops.mesh_simplify) on the GPU over the meshes of tools/time_mesh_components.py.
Prints one JSON line per case and target, and one with the device name and power limit.

    python tools/time_mesh_simplify.py [--reps 2] [--cases dense256,dense512,sparse1024,sparse2048] [--oracle]

Each case's mesh (the sphere and balls field, dense marching cubes at res 256 / 512, sparse at res 1024 / 2048) is
simplified to 10 % and to 1 % of its faces.  Per target: the best and median of --reps sync'd wall-clock times of
ops.mesh_simplify (id check, init, every round with its read-back of {F_live, collapses}, emit), the rounds, the time
per round and the faces.  --oracle also times the NumPy oracle (tests/simplify_oracle.py) on a small mesh, the only
host comparison: no host decimator is installed.
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

from sparf_b200 import ops
from time_density import power_limit
from time_mesh_components import dense_volume, sparse_blocks, timed


def mesh_of(name):
    kind = "dense" if name.startswith("dense") else "sparse"
    res = int(name[len(kind):])
    if kind == "dense":
        return ops.marching_cubes(dense_volume(res), 0.0)
    sigma, slots, ids = sparse_blocks(res)
    return ops.marching_cubes_sparse(sigma, res, slots, ids, 0.0)


def run_case(name, reps):
    verts, faces = mesh_of(name)
    torch.cuda.empty_cache()
    F = faces.shape[0]
    for frac in (0.1, 0.01):
        target = int(F * frac)
        st = {}
        ops.mesh_simplify(verts, faces, target, stats=st)         # warm-up
        (v, f, _, _), t = timed(lambda: ops.mesh_simplify(verts, faces, target), reps)
        print(json.dumps(dict(case=name, V=verts.shape[0], F=F, target=target, F_out=f.shape[0], V_out=v.shape[0],
                              rounds=st["rounds"], collapses=st["collapses"], simplify=t,
                              ms_per_round=round(t["best_ms"] / max(st["rounds"], 1), 3))), flush=True)


def run_oracle():
    import simplify_oracle as SO
    verts, faces = ops.marching_cubes(dense_volume(32), 0.0)
    target = faces.shape[0] // 10
    v, f = verts.cpu().numpy(), faces.cpu().numpy()
    t = time.perf_counter()
    ref = SO.simplify(v, f, target)
    t_host = (time.perf_counter() - t) * 1e3
    ops.mesh_simplify(verts, faces, target)
    (vo, fo, _, _), t_dev = timed(lambda: ops.mesh_simplify(verts, faces, target), 3)
    assert torch.equal(fo.cpu(), torch.from_numpy(ref[1])) and torch.equal(vo.cpu(), torch.from_numpy(ref[0]))
    print(json.dumps(dict(case="oracle_dense32", F=faces.shape[0], target=target, F_out=fo.shape[0], rounds=ref[4],
                          host_oracle_ms=round(t_host, 1), simplify=t_dev)), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--cases", default="dense256,dense512,sparse1024,sparse2048")
    ap.add_argument("--oracle", action="store_true", help="also time the NumPy oracle on a small mesh")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "time_mesh_simplify.py runs on a GPU"
    print(json.dumps(dict(device=torch.cuda.get_device_name(), power_limit_w=power_limit())), flush=True)
    if args.oracle:
        run_oracle()
    for name in args.cases.split(","):
        run_case(name, args.reps)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
