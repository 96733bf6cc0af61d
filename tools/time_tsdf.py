#!/usr/bin/env python
"""Time TSDF fusion (sparf_b200/tsdf.py) on the GPU.  Prints one JSON line with the device name and power limit.

    python tools/time_tsdf.py [--reps 10]

(a) tsdf.integrate_ of 60 views of 300 x 400 pixels (exact depth maps of a sphere of radius 0.6 from cameras around the
    box, constant colour, every pixel valid) into volumes of res 256 and 512 over [-1.2, 1.2]^3: CUDA events around
    one call, best and median of --reps after a warm-up.  Bytes: the volume's state read and written once (40 B per
    lattice point) plus the maps read once (17 B per pixel); GB/s = bytes / time, against the H100 SXM's 3.35 TB/s.
(b) tsdf.fuse_renders on a DTU-shaped setting: 3 views of 300 x 400 pixels, 128 coarse + 128 fine samples (the shapes of
    golden case c2_hier), the octahedron scene of tools/time_occupancy.py, into a res-256 volume; the renders and the
    integration timed apart (tsdf.render_batches), plus masked marching cubes of the result.
"""
import argparse
import json
import math
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "golden"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np
import torch

import common
from sparf_b200 import ops, tsdf
from time_density import power_limit
from time_occupancy import octahedron_graph, sync_ms

HBM_BYTES_PER_S = 3.35e12


def ring(B, H, W, radius=3.0, focal=None):
    poses = []
    for b in range(B):
        a = 2 * math.pi * b / B
        poses.append(common.look_at_w2c((radius * math.sin(a), 0.8 * math.sin(3 * a), -radius * math.cos(a))))
    f = float(focal if focal is not None else 1.1 * max(H, W))
    K = np.array([[f, 0, W / 2.0], [0, f, H / 2.0], [0, 0, 1]], np.float32)
    return torch.from_numpy(np.stack(poses)).cuda(), torch.from_numpy(np.stack([K] * B)).cuda()


def sphere_depth(pose, K, H, W, r=0.6, far=100.0):
    o, d = ops.raygen(pose, K, W, ray_idx=torch.arange(H * W, device="cuda"))
    o, d = o.double(), d.double()
    a, b, c = (d * d).sum(-1), 2 * (o * d).sum(-1), (o * o).sum(-1) - r * r
    disc = b * b - 4 * a * c
    t = (-b - disc.clamp_min(0).sqrt()) / (2 * a)
    return torch.where((disc > 0) & (t > 0), t, torch.full_like(t, far)).float().view(-1, H, W).contiguous()


def event_ms(fn, reps):
    fn()
    times = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1))
    return min(times), float(np.median(times))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "time_tsdf.py measures on a GPU"
    out = dict(device=torch.cuda.get_device_name(), power_limit_w=power_limit())
    B, H, W = 60, 300, 400
    pose, K = ring(B, H, W)
    depth = sphere_depth(pose, K, H, W)
    rgb = torch.full((B, H, W, 3), 0.5, device="cuda")
    valid = torch.ones(B, H, W, dtype=torch.bool, device="cuda")
    for res in (256, 512):
        vol = tsdf.TSDFVolume(res=res)
        best, med = event_ms(lambda: tsdf.integrate_(vol, depth, pose, K, rgb=rgb, valid=valid), args.reps)
        n3 = vol.n ** 3
        nbytes = 40 * n3 + 17 * B * H * W
        out["integrate_res%d" % res] = dict(views=B, H=H, W=W, lattice_points=n3, ms=round(best, 3), ms_median=round(med, 3),
                                            gb_per_s=round(nbytes / best / 1e6, 1),
                                            hbm_fraction=round(nbytes / (best * 1e-3) / HBM_BYTES_PER_S, 3),
                                            ns_per_point_view=round(best * 1e6 / (n3 * B), 4))
        del vol

    ops.set_engine("tc_3x" if ops._lib.lib().sparf_engine_available(ops._lib.ENGINE_TC_3X) else "auto")
    B, H, W = 3, 300, 400
    opt = common.make_opt(S=128, S_fine=128, fine=True, depth_range=(1.5, 4.5))
    data = common.make_scene(3, B, H, W, focal=800.0)
    pose, K = data.pose.cuda(), data.intr.cuda()
    with torch.no_grad():
        net = octahedron_graph(opt, 0.6)
        vol = tsdf.TSDFVolume(res=256)
        runs = []
        for rep in range(args.reps // 2 + 2):
            vol.reset_()
            torch.cuda.synchronize()
            t = dict(render_ms=0.0, integrate_ms=0.0)
            batches = tsdf.render_batches(opt, net, pose, K, H, W, (1.5, 4.5), device="cuda")
            while True:
                ms, batch = sync_ms(lambda: next(batches, None))
                t["render_ms"] += ms
                if batch is None:
                    break
                t["integrate_ms"] += sync_ms(lambda: tsdf.integrate_(vol, batch[0], batch[1], batch[2], rgb=batch[3],
                                                                    valid=batch[4]))[0]
            t["fuse_ms"] = sync_ms(lambda: tsdf.fuse_renders(opt, net, vol.reset_(), pose, K, H, W, (1.5, 4.5)))[0]
            t["marching_cubes_ms"], m = sync_ms(lambda: tsdf.extract_mesh(vol))
            if rep:                     # rep 0 warms up
                runs.append(t)
        best = {k: round(min(r[k] for r in runs), 2) for k in runs[0]}
        out["fuse_renders_dtu"] = dict(views=B, H=H, W=W, samples="128+128", res=256, V=m["vertices"].shape[0],
                                       F=m["faces"].shape[0], observed_points=int(vol.weight.gt(0).sum().item()), **best)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
