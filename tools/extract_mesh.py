#!/usr/bin/env python
"""Extract a mesh from a reference-format snapshot and write it as a binary PLY (sparf_b200.mesh: BARF's recipe over
opt.trimesh, on the GPU).

    python tools/extract_mesh.py model.pth.tar --out mesh.ply [--network nerf|nerf_fine] [--res 128]
                                 [--range -1.2 1.2] [--thres 25] [--normals] [--barf-c2f START END] [--sparse]
    python tools/extract_mesh.py model.pth.tar --out mesh.ply --tsdf cameras.npz [--res 128] [--range -1.2 1.2]
                                 [--trunc T] [--samples 128] [--samples-fine 128] [--barf-c2f START END]

The snapshot is what the reference's trainer saves (base_trainer.py:196-216): the model dict is ckpt["state_dict"],
with the Graph's keys nerf.* / nerf_fine.* (or, from a joint pose trainer, those under "nerf_net").  The architecture
is read from the tensor shapes.  The BARF mask applies at the snapshot's progress when --barf-c2f gives the schedule
the model was trained with.  --sparse extracts with mesh.extract_mesh_sparse's phases (the density only in the 8^3-cell
blocks near the surface; for high resolutions) and also prints the active-block count and the points evaluated.
--tsdf CAMERAS fuses renders instead (sparf_b200.tsdf): a Graph with both networks of the snapshot (the fine one when
present) renders the views of CAMERAS, a .npz or .pt file with pose_w2c [B,3,4], intr [B,3,3], H, W and depth_range [2]
(metric near, far), with --samples / --samples-fine samples per ray; the depth and colour maps are integrated into a TSDF
volume over --res / --range with truncation --trunc (default tsdf.TRUNC_VOXELS voxels), and the coloured mesh of its
zero level is written.
Prints V, F and the time of each phase.
"""
import argparse
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
import torch


def opt_from_state_dict(sd, barf_c2f=None):
    """The options a NeRF with these tensors was built from (frequency_nerf.py:87-134)"""
    from sparf_b200.utils.edict import edict
    n = len({k.split(".")[1] for k in sd if k.startswith("mlp_feat.")})
    w0 = sd["mlp_feat.0.weight"]
    width, in3 = w0.shape[0], w0.shape[1]
    skip = [i for i in range(1, n) if sd["mlp_feat.%d.weight" % i].shape[1] == width + in3]
    head = sd["mlp_rgb.0.weight"]
    opt = edict()
    opt.arch = edict(layers_feat=[None] + [width] * n, layers_feat_fine=None, layers_rgb=[None, head.shape[0], 3], skip=skip,
                     density_activ="softplus", tf_init=True,
                     posenc=edict(include_pi_in_posenc=True, add_raw_3D_points=True, add_raw_rays=True, log_sampling=True,
                                  L_3D=(in3 - 3) // 6, L_view=(head.shape[1] - width - 3) // 6))
    opt.nerf = edict(view_dep=True)
    opt.barf_c2f = list(barf_c2f) if barf_c2f else None
    return opt


def graph_opt_from_state_dict(sd, barf_c2f, depth_range, samples, samples_fine):
    """The options of a Graph with the networks of a snapshot's state dict (keys nerf.* and, if present, nerf_fine.*) that
    renders metric-depth views deterministically (val mode) with the given samples per ray"""
    from sparf_b200.utils.edict import edict
    opt = opt_from_state_dict({k[len("nerf."):]: v for k, v in sd.items() if k.startswith("nerf.")}, barf_c2f)
    fine = any(k.startswith("nerf_fine.") for k in sd)
    opt.nerf = edict(view_dep=True, depth=edict(param="metric", range=[float(x) for x in depth_range]),
                     sample_intvs=samples, sample_stratified=False, fine_sampling=fine, sample_intvs_fine=samples_fine,
                     rand_rays=1024, density_noise_reg=False, setbg_opaque=False)
    opt.camera = edict(model="perspective", ndc=False)
    opt.mask_img, opt.max_iter = False, 1
    return opt


def load_cameras(path):
    """pose_w2c [B,3,4], intr [B,3,3] (fp32 tensors), H, W, depth_range (near, far) of a .npz or .pt camera file"""
    import numpy as np
    if path.endswith(".npz"):
        with np.load(path) as z:
            cams = {k: z[k] for k in z.files}
    else:
        cams = torch.load(path, map_location="cpu", weights_only=False)
    t = lambda x: torch.as_tensor(np.asarray(x), dtype=torch.float32)
    return (t(cams["pose_w2c"]), t(cams["intr"]), int(cams["H"]), int(cams["W"]),
            tuple(float(x) for x in np.asarray(cams["depth_range"]).reshape(2)))


def main_tsdf(args):
    from sparf_b200 import mesh, tsdf
    from sparf_b200.renderer import Graph
    t0 = time.perf_counter()
    sd = torch.load(args.snapshot, map_location="cpu", weights_only=False)["state_dict"]
    sd = sd.get("nerf_net", sd)
    assert any(k.startswith("nerf.") for k in sd), "the snapshot has no nerf.* tensors"
    pose, intr, H, W, depth_range = load_cameras(args.tsdf)
    opt = graph_opt_from_state_dict(sd, args.barf_c2f, depth_range, args.samples, args.samples_fine)
    graph = Graph(opt, torch.device("cuda"))
    graph.load_state_dict({k: v for k, v in sd.items() if k.startswith(("nerf.", "nerf_fine."))})
    vol = tsdf.TSDFVolume(res=args.res, range=args.range, trunc=args.trunc)
    phases = {"load": time.perf_counter() - t0}

    def phase(name, fn):
        torch.cuda.synchronize()
        t = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        phases[name] = phases.get(name, 0.0) + time.perf_counter() - t
        return out

    # tsdf.fuse_renders, with the renders and the integrations timed apart
    batches = tsdf.render_batches(opt, graph, pose, intr, H, W, depth_range, device=vol.tsdf.device)
    while True:
        batch = phase("render", lambda: next(batches, None))
        if batch is None:
            break
        phase("integrate", lambda: tsdf.integrate_(vol, batch[0], batch[1], batch[2], rgb=batch[3], valid=batch[4]))
    m = phase("marching_cubes", lambda: tsdf.extract_mesh(vol))
    phase("write_ply", lambda: mesh.write_ply(args.out, m["vertices"], m["faces"], colors=m["colors"]))
    print("%s: V %d, F %d (TSDF of %d views %dx%d, res %d, range %s, trunc %g)"
          % (args.out, m["vertices"].shape[0], m["faces"].shape[0], pose.shape[0], H, W, vol.res, list(vol.range),
             vol.trunc))
    print("  " + ", ".join("%s %.3f s" % kv for kv in phases.items()))


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("snapshot")
    ap.add_argument("--out", required=True)
    ap.add_argument("--network", default="nerf", choices=["nerf", "nerf_fine"])
    ap.add_argument("--res", type=int, default=128)
    ap.add_argument("--range", type=float, nargs=2, default=[-1.2, 1.2])
    ap.add_argument("--thres", type=float, default=25.0)
    ap.add_argument("--normals", action="store_true")
    ap.add_argument("--barf-c2f", type=float, nargs=2, default=None)
    ap.add_argument("--sparse", action="store_true", help="evaluate only the blocks near the surface (res: multiple of 8)")
    ap.add_argument("--tsdf", metavar="CAMERAS", default=None, help="fuse renders of these cameras (.npz / .pt) instead")
    ap.add_argument("--trunc", type=float, default=None, help="TSDF truncation in world units (--tsdf)")
    ap.add_argument("--samples", type=int, default=128, help="coarse samples per ray of the renders (--tsdf)")
    ap.add_argument("--samples-fine", type=int, default=128, help="fine samples per ray of the renders (--tsdf)")
    args = ap.parse_args(argv)
    assert torch.cuda.is_available(), "extract_mesh.py runs on a GPU"
    if args.tsdf:
        return main_tsdf(args)
    from sparf_b200 import mesh
    from sparf_b200.frequency_nerf import NeRF
    from sparf_b200.utils.edict import edict

    t0 = time.perf_counter()
    sd = torch.load(args.snapshot, map_location="cpu", weights_only=False)["state_dict"]
    sd = sd.get("nerf_net", sd)
    prefix = args.network + "."
    sd = {k[len(prefix):]: v for k, v in sd.items() if k.startswith(prefix)}
    assert sd, "the snapshot has no %s.* tensors" % args.network
    opt = opt_from_state_dict(sd, args.barf_c2f)
    opt.trimesh = edict(res=args.res, range=list(args.range), thres=args.thres)
    nerf = NeRF(opt).cuda()
    nerf.load_state_dict(sd)
    res, rng, thres = mesh.trimesh_settings(opt)
    phases = {}

    def phase(name, fn):
        torch.cuda.synchronize()
        t = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        phases[name] = time.perf_counter() - t
        return out

    phases["load"] = time.perf_counter() - t0
    if args.sparse:
        from sparf_b200 import ops
        mesh.check_sparse_res(res)
        axis = mesh.lattice_axis(res, rng)
        coarse = phase("coarse", lambda: mesh.coarse_density(nerf, axis))
        slots, ids = phase("classify", lambda: ops.mcubes_sparse_classify(coarse, thres))
        sigma = phase("fine", lambda: mesh.block_density(nerf, axis, ids))
        verts, faces = phase("marching_cubes", lambda: ops.marching_cubes_sparse(sigma, res, slots, ids, thres))
        nb = res // mesh.BLOCK
        print("active blocks %d of %d, points evaluated %d (dense lattice %d)"
              % (ids.numel(), nb ** 3, coarse.numel() + sigma.numel(), (res + 1) ** 3))
    else:
        sigma = phase("density_grid", lambda: mesh.density_grid(opt, nerf))
        verts, faces = phase("marching_cubes", lambda: mesh.marching_cubes(sigma, thres))
    del sigma
    verts = mesh.to_world(verts, res, rng)
    normals = phase("normals", lambda: mesh.density_normals(nerf, verts)) if args.normals else None
    phase("write_ply", lambda: mesh.write_ply(args.out, verts, faces, normals))
    print("%s: V %d, F %d (res %d, range %s, thres %g)" % (args.out, verts.shape[0], faces.shape[0], res, list(rng), thres))
    print("  " + ", ".join("%s %.3f s" % kv for kv in phases.items()))


if __name__ == "__main__":
    main()
