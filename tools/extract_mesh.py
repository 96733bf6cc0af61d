#!/usr/bin/env python
"""Extract a mesh from a reference-format snapshot and write it as a binary PLY (sparf_b200.mesh: BARF's recipe over
opt.trimesh, on the GPU).

    python tools/extract_mesh.py model.pth.tar --out mesh.ply [--network nerf|nerf_fine] [--res 128]
                                 [--range -1.2 1.2] [--thres 25] [--normals] [--barf-c2f START END] [--sparse]

The snapshot is what the reference's trainer saves (base_trainer.py:196-216): the model dict is ckpt["state_dict"],
with the Graph's keys nerf.* / nerf_fine.* (or, from a joint pose trainer, those under "nerf_net").  The architecture
is read from the tensor shapes.  The BARF mask applies at the snapshot's progress when --barf-c2f gives the schedule
the model was trained with.  --sparse extracts with mesh.extract_mesh_sparse's phases (the density only in the 8^3-cell
blocks near the surface; for high resolutions) and also prints the active-block count and the points evaluated.
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
    args = ap.parse_args(argv)
    assert torch.cuda.is_available(), "extract_mesh.py runs on a GPU"
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
