#!/usr/bin/env python
"""Time mesh extraction (sparf_b200.mesh) on the GPU: density_grid over BARF's lattice, and marching cubes split into
count, the totals' copy to the host, and emit.  Prints one JSON line with the device name and power limit.

    python tools/time_mesh.py [--res 128,256,512] [--engine tc_3x]

Network: the synthetic teacher of tools/train_synthetic.py (common.det_weights(opt, 5, peaky=True, sigma_bias=-2.0)).
Iso value: the 90th percentile of the lattice's density, so that the mesh is large.  Per resolution:
  * density_grid_ms, and explicit_points_ms: ops.density_forward(features=False) + softplus over the same points held
    as materialised arrays in the same slabs (the lattice built slab-wise costs nothing extra if the two agree);
  * mc_count_ms, mc_emit_ms (CUDA events), mc_sync_ms (host time of the totals' copy), mc_total_ms (host, one call);
  * mc_bytes: what the kernels must move, counted from shapes (count: the volume once, 8 B per point of offsets out;
    emit: the volume and the offsets once, 12 B per vertex and 24 B per face out), and mc_gb_per_s over count + emit.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "golden")):
    sys.path.insert(0, p)
import ctypes

import torch

import common
from sparf_b200 import _lib, mesh, ops
from sparf_b200.frequency_nerf import NeRF
from time_density import power_limit


def events_ms(fn, reps=1):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def time_mc(sigma, iso, reps):
    """(count ms, totals copy ms, emit ms, host ms of a whole ops.marching_cubes call, V, F)"""
    L = _lib.lib()
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    nx, ny, nz = sigma.shape
    ws = torch.empty(L.sparf_mcubes_workspace_bytes(nx, ny, nz), dtype=torch.uint8, device="cuda")
    totals = torch.empty(2, dtype=torch.int64, device="cuda")
    st = ops._stream()
    count = lambda: _lib.check(L.sparf_mcubes_count(p(sigma), nx, ny, nz, iso, p(totals), p(ws), ws.numel(), st), "count")
    count()
    torch.cuda.synchronize()
    t = time.perf_counter()
    V, F = totals.tolist()
    sync_ms = (time.perf_counter() - t) * 1e3       # the copy alone (the device is idle)
    verts = torch.empty(V, 3, device="cuda")
    faces = torch.empty(F, 3, dtype=torch.int64, device="cuda")
    emit = lambda: _lib.check(L.sparf_mcubes_emit(p(sigma), nx, ny, nz, iso, p(verts), p(faces), p(ws), ws.numel(), st), "emit")
    emit()
    count_ms = events_ms(count, reps)
    emit_ms = events_ms(emit, reps)
    ops.marching_cubes(sigma, iso)
    torch.cuda.synchronize()
    t = time.perf_counter()
    ops.marching_cubes(sigma, iso)
    torch.cuda.synchronize()
    return count_ms, sync_ms, emit_ms, (time.perf_counter() - t) * 1e3, V, F


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--res", default="128,256,512")
    ap.add_argument("--engine", default="tc_3x")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "time_mesh.py measures on a GPU"
    opt = common.make_opt()
    nerf = NeRF(opt).cuda()
    nerf.load_state_dict({k: v.cuda() for k, v in common.det_weights(opt, 5, peaky=True, sigma_bias=-2.0).items()})
    eng = _lib.ENGINES[args.engine]
    out = dict(device=torch.cuda.get_device_name(), power_limit_w=power_limit(), engine=args.engine, hbm_peak_tb_s=3.35)
    spec, trunk, prog = nerf._spec(), mesh._trunk(nerf), nerf.progress.detach()
    with torch.no_grad():
        for res in [int(r) for r in args.res.split(",")]:
            n = res + 1
            grid = lambda: mesh.density_grid(opt, nerf, res=res, engine=eng)
            sigma = grid()                                                    # warm-up (every slab shape)
            t = mesh.lattice_axis(res, mesh.TRIMESH_DEFAULTS["range"]).cuda()
            slabs = [pts.clone() for _, pts in mesh.lattice_slabs(t, max(1, mesh.SLAB_POINTS // (n * n)))]
            dens = torch.empty(n ** 3, device="cuda")

            def explicit():
                o = 0
                for pts in slabs:
                    raw, _ = ops.density_forward(spec, pts, trunk, progress=prog, engine=eng, features=False)
                    dens[o:o + raw.shape[0]] = torch.nn.functional.softplus(raw)
                    o += raw.shape[0]

            explicit()
            torch.cuda.synchronize()
            r = dict(points=n ** 3)
            g_ms, x_ms = [], []
            for _ in range(3):                  # alternated, best of three
                g_ms.append(events_ms(grid))
                x_ms.append(events_ms(explicit))
            r["density_grid_ms"], r["explicit_points_ms"] = min(g_ms), min(x_ms)
            r["same_values"] = bool(torch.equal(dens.view(n, n, n), sigma))
            r["density_grid_mpts_per_s"] = n ** 3 / r["density_grid_ms"] / 1e3
            del slabs
            iso = torch.quantile(sigma.view(-1)[::97].float(), 0.9).item()
            reps = 20 if res <= 256 else 5
            c_ms, s_ms, e_ms, tot_ms, V, F = time_mc(sigma, iso, reps)
            nbytes = (4 + 8) * n ** 3 + (4 + 8) * n ** 3 + 12 * V + 24 * F
            r.update(iso=iso, V=V, F=F, mc_count_ms=c_ms, mc_sync_ms=s_ms, mc_emit_ms=e_ms, mc_total_ms=tot_ms,
                     mc_bytes=nbytes, mc_gb_per_s=nbytes / ((c_ms + e_ms) * 1e-3) / 1e9)
            out["res%d" % res] = r
            del sigma, dens
            torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
