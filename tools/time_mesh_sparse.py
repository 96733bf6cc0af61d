#!/usr/bin/env python
"""Time sparse mesh extraction (mesh.extract_mesh_sparse) against the dense one (mesh.extract_mesh) on the GPU.  Prints
one JSON line with the device name and power limit.

    python tools/time_mesh_sparse.py [--res 256,512,1024] [--sparse-only 2048] [--engine tc_3x] [--reps 2]

Scene: the octahedron NeRF of time_occupancy.octahedron_weights (σ = softplus(c - k |x|_1), radius 0.6, k = 40) over
BARF's default range [-1.2, 1.2], iso 1.  Per resolution in --res, dense and sparse are run alternately --reps times
(best of each, host clock around synchronised phases):
  * dense: density_grid_ms, mc_ms (ops.marching_cubes), total_ms;
  * sparse: coarse_ms, classify_ms, fine_ms (density of the active blocks), mc_ms (ops.marching_cubes_sparse, with the
    vertex sort), total_ms; active_fraction, points_evaluated, V, F, and whether the mesh equals the dense one;
and for --sparse-only the sparse phases alone with the peak device memory of the call.
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

import torch

import common
from sparf_b200 import mesh, ops
from sparf_b200.frequency_nerf import NeRF
from time_density import power_limit
from time_occupancy import octahedron_weights

RADIUS, K, ISO, RANGE = 0.6, 40.0, 1.0, (-1.2, 1.2)


def timed(phases, name, fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    phases[name] = (time.perf_counter() - t) * 1e3
    return out


def dense(nerf, res):
    ph = {}
    axis = mesh.lattice_axis(res, RANGE)
    sigma = timed(ph, "density_grid_ms", lambda: mesh.lattice_density(nerf, axis))
    v, f = timed(ph, "mc_ms", lambda: ops.marching_cubes(sigma, ISO))
    del sigma
    ph["total_ms"] = ph["density_grid_ms"] + ph["mc_ms"]
    return ph, (v, f)


def sparse(nerf, res):
    ph = {}
    axis = mesh.lattice_axis(res, RANGE)
    coarse = timed(ph, "coarse_ms", lambda: mesh.coarse_density(nerf, axis))
    slots, ids = timed(ph, "classify_ms", lambda: ops.mcubes_sparse_classify(coarse, ISO))
    sigma = timed(ph, "fine_ms", lambda: mesh.block_density(nerf, axis, ids))
    v, f = timed(ph, "mc_ms", lambda: ops.marching_cubes_sparse(sigma, res, slots, ids, ISO))
    ph["total_ms"] = ph["coarse_ms"] + ph["classify_ms"] + ph["fine_ms"] + ph["mc_ms"]
    nb = res // mesh.BLOCK
    ph.update(active_blocks=ids.numel(), active_fraction=ids.numel() / nb ** 3,
              points_evaluated=coarse.numel() + sigma.numel(), dense_points=(res + 1) ** 3, V=v.shape[0], F=f.shape[0])
    return ph, (v, f)


def best(runs):
    out = dict(runs[0])
    for k in out:
        if k.endswith("_ms"):
            out[k] = min(r[k] for r in runs)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--res", default="256,512,1024")
    ap.add_argument("--sparse-only", default="2048")
    ap.add_argument("--engine", default="tc_3x")
    ap.add_argument("--reps", type=int, default=2)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "time_mesh_sparse.py measures on a GPU"
    ops.set_engine(args.engine)
    opt = common.make_opt()
    nerf = NeRF(opt).cuda()
    nerf.load_state_dict({k: v.cuda() for k, v in octahedron_weights(opt, c=K * RADIUS, k=K).items()})
    out = dict(device=torch.cuda.get_device_name(), power_limit_w=power_limit(), engine=args.engine, iso=ISO)
    with torch.no_grad():
        dense(nerf, 64), sparse(nerf, 64)                          # module loads, first launches
        for res in [int(r) for r in args.res.split(",") if r]:
            d_runs, s_runs = [], []
            for _ in range(args.reps):                              # alternated
                ph, dm = dense(nerf, res)
                d_runs.append(ph)
                del dm
                torch.cuda.empty_cache()
                ph, sm = sparse(nerf, res)
                s_runs.append(ph)
            ph, dm = dense(nerf, res)
            same = bool(torch.equal(dm[1], sm[1]) and torch.equal(dm[0].view(torch.int32), sm[0].view(torch.int32)))
            dV, dF = dm[0].shape[0], dm[1].shape[0]
            del dm, sm
            torch.cuda.empty_cache()
            d, s = best(d_runs), best(s_runs)
            out["res%d" % res] = dict(dense=d, sparse=s, dense_V=dV, dense_F=dF, same_mesh=same,
                                      speedup=d["total_ms"] / s["total_ms"])
        for res in [int(r) for r in args.sparse_only.split(",") if r]:
            torch.cuda.empty_cache()
            torch.cuda.reset_peak_memory_stats()
            ph, _ = sparse(nerf, res)
            ph["peak_mem_gb"] = torch.cuda.max_memory_allocated() / 1e9
            out["sparse_res%d" % res] = ph
    print(json.dumps(out))


if __name__ == "__main__":
    main()
