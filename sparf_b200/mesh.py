"""Mesh extraction from a trained NeRF, BARF's recipe on the device: the density on the lattice of `opt.trimesh`
(train_settings/default_config.py:267-271), marching cubes (csrc/mcubes.cu), world coordinates, optional normals from
the density's gradient, and a binary PLY writer.

    from sparf_b200 import mesh
    m = mesh.extract_mesh(opt, graph.nerf, normals=True)        # or graph.nerf_fine
    mesh.write_ply("scene.ply", m["vertices"], m["faces"], m["normals"])
"""
from __future__ import annotations

import numpy as np
import torch

from . import _lib, ops

# train_settings/default_config.py:267-271, used where `opt` has no `trimesh` entry
TRIMESH_DEFAULTS = dict(res=128, range=(-1.2, 1.2), thres=25.0)
SLAB_POINTS = 1 << 22       # lattice points per density_forward call
NORMAL_CHUNK = 1 << 18      # vertices per density backward call


def trimesh_settings(opt, res=None, range=None, thres=None):
    """(res, (r0, r1), thres): the arguments where given, else opt.trimesh's, else TRIMESH_DEFAULTS"""
    tm = opt.get("trimesh") if isinstance(opt, dict) else getattr(opt, "trimesh", None)
    tm = tm or {}
    res = int(res if res is not None else tm.get("res", TRIMESH_DEFAULTS["res"]))
    r0, r1 = range if range is not None else tm.get("range", TRIMESH_DEFAULTS["range"])
    thres = float(thres if thres is not None else tm.get("thres", TRIMESH_DEFAULTS["thres"]))
    return res, (float(r0), float(r1)), thres


def lattice_axis(res: int, range) -> torch.Tensor:
    """BARF's lattice coordinates torch.linspace(r0, r1, res + 1) in fp32, computed on the host (the same values on any
    device)"""
    return torch.linspace(float(range[0]), float(range[1]), res + 1, dtype=torch.float32)


def lattice_slabs(t: torch.Tensor, rows: int):
    """The lattice stack(meshgrid(t, t, t, indexing="ij"), -1) (axis 0 = x) in slabs of `rows` x-planes: yields (i0,
    points [rows * n * n, 3]) without materialising the whole lattice"""
    for i0 in range(0, t.numel(), rows):
        ts = t[i0:i0 + rows]
        yield i0, torch.stack(torch.meshgrid(ts, t, t, indexing="ij"), dim=-1).reshape(-1, 3)


def _engine(engine):
    return None if engine is None else (_lib.ENGINES[engine] if isinstance(engine, str) else int(engine))


def _trunk(nerf):
    return [p.detach() for p in nerf.kernel_params()[:2 * len(nerf.mlp_feat)]]


@torch.no_grad()
def density_grid(opt, nerf, res=None, range=None, engine=None) -> torch.Tensor:
    """sigma [res+1, res+1, res+1] on nerf's device: softplus of the raw density (ops.density_forward, features=False; no
    noise, the BARF mask at nerf.progress) at BARF's lattice points (lattice_axis; axis 0 = x), evaluated slab by slab
    so that the point array of the whole lattice never exists.  res / range default to opt.trimesh (TRIMESH_DEFAULTS
    where opt has none).  The reference's trimesh.chunk_size is a memory setting of its PyTorch evaluation and is not
    used: the slabs and the kernels' own chunking bound the memory here.  engine: None = the current ops engine."""
    res, rng, _ = trimesh_settings(opt, res, range)
    return lattice_density(nerf, lattice_axis(res, rng), engine=engine)


@torch.no_grad()
def lattice_density(nerf, axis: torch.Tensor, engine=None, warp=None) -> torch.Tensor:
    """sigma [n, n, n] (n = axis.numel()) on nerf's device: softplus of the raw density (ops.density_forward,
    features=False; no noise, the BARF mask at nerf.progress) at the lattice points of lattice_slabs(axis), slab by slab.
    warp: None (the lattice points are world points), or a map of one slab's lattice points [P, 3] to (world points
    [P, 3], a bool [P] mask of the points that are not evaluated and get sigma = NaN, or None)."""
    dev = nerf.progress.device
    t = axis.to(dev)
    n = t.numel()
    sigma = torch.empty(n, n, n, device=dev, dtype=torch.float32)
    spec, trunk = nerf._spec(), _trunk(nerf)
    for i0, pts in lattice_slabs(t, max(1, SLAB_POINTS // (n * n))):
        rows = pts.shape[0] // (n * n)
        skip = None
        if warp is not None:
            pts, skip = warp(pts)
        raw, _ = ops.density_forward(spec, pts, trunk, progress=nerf.progress.detach(), engine=_engine(engine),
                                     features=False)
        s = torch.nn.functional.softplus(raw)
        if skip is not None:
            s = s.masked_fill(skip.view(s.shape), float("nan"))
        sigma[i0:i0 + rows] = s.view(-1, n, n)
    return sigma


def marching_cubes(volume: torch.Tensor, isovalue: float):
    """(verts [V, 3] fp32 in index space, faces [F, 3] int64) of the iso-surface {volume >= isovalue}: ops.marching_cubes"""
    return ops.marching_cubes(volume, isovalue)


def to_world(verts: torch.Tensor, res: int, range) -> torch.Tensor:
    """index space -> world: BARF's verts / res * (r1 - r0) + r0"""
    r0, r1 = range
    return verts / res * (r1 - r0) + r0


@torch.no_grad()
def density_normals(nerf, points: torch.Tensor, engine=None) -> torch.Tensor:
    """-grad(raw) / |grad(raw)| at points [M, 3] (the direction of falling density), 0 where the gradient is 0; the
    point gradient (ops.density_gradient, no weight gradients) in chunks of NORMAL_CHUNK points"""
    spec, trunk = nerf._spec(), _trunk(nerf)
    out = torch.empty_like(points)
    for c0 in range(0, points.shape[0], NORMAL_CHUNK):
        g = ops.density_gradient(spec, points[c0:c0 + NORMAL_CHUNK], trunk, progress=nerf.progress.detach(),
                                 engine=_engine(engine))
        out[c0:c0 + NORMAL_CHUNK] = unit_normals(g)
    return out


def unit_normals(g: torch.Tensor) -> torch.Tensor:
    """-g / |g| over the last axis, 0 where |g| = 0: the normal of a density gradient g [..., 3]"""
    norm = g.norm(dim=-1, keepdim=True)
    return torch.where(norm > 0, -g / norm, torch.zeros_like(g))


def extract_mesh(opt, nerf, normals: bool = False, engine=None) -> dict:
    """BARF's mesh extraction for one network (graph.nerf or graph.nerf_fine): density_grid over opt.trimesh, marching
    cubes at opt.trimesh.thres, world vertices by BARF's formula (to_world).  -> dict(vertices [V, 3] fp32, faces [F, 3]
    int64[, normals [V, 3]]) on nerf's device."""
    res, rng, thres = trimesh_settings(opt)
    verts, faces = marching_cubes(density_grid(opt, nerf, engine=engine), thres)
    out = dict(vertices=to_world(verts, res, rng), faces=faces)
    if normals:
        out["normals"] = density_normals(nerf, out["vertices"], engine=engine)
    return out


BLOCK = _lib.MCUBES_BLOCK       # cells per block edge of extract_mesh_sparse


def check_sparse_res(res: int) -> None:
    if res < BLOCK or res % BLOCK:
        raise ValueError("sparse mesh extraction needs res to be a positive multiple of %d (got %d)" % (BLOCK, res))


@torch.no_grad()
def coarse_density(nerf, axis: torch.Tensor, engine=None) -> torch.Tensor:
    """sigma [nb+1]^3 at the lattice points whose indices are all multiples of BLOCK: lattice_density over axis[::BLOCK],
    so the values are density_grid's at those points bit for bit"""
    return lattice_density(nerf, axis[::BLOCK], engine=engine)


@torch.no_grad()
def block_density(nerf, axis: torch.Tensor, block_ids: torch.Tensor, engine=None) -> torch.Tensor:
    """sigma [n_active, 9, 9, 9] at the points of the given blocks (ops.mcubes_sparse_points), in slabs of about
    SLAB_POINTS points; each point is evaluated as density_grid evaluates it (same fp32 input, rows independent)"""
    dev = nerf.progress.device
    t = axis.to(dev)
    P = BLOCK + 1
    n = block_ids.numel()
    sigma = torch.empty(n, P, P, P, device=dev, dtype=torch.float32)
    spec, trunk = nerf._spec(), _trunk(nerf)
    per = max(1, SLAB_POINTS // P ** 3)
    for b0 in range(0, n, per):
        nblk = min(per, n - b0)
        pts = ops.mcubes_sparse_points(t, block_ids, b0, nblk)
        raw, _ = ops.density_forward(spec, pts, trunk, progress=nerf.progress.detach(), engine=_engine(engine),
                                     features=False)
        sigma[b0:b0 + nblk] = torch.nn.functional.softplus(raw).view(nblk, P, P, P)
    return sigma


def extract_mesh_sparse(opt, nerf, normals: bool = False, engine=None, stats=None) -> dict:
    """extract_mesh for high lattice resolutions: the density only in the 8^3-cell blocks near the surface.  A coarse pass
    over every 8th lattice point marks the active blocks (include/sparf_b200.h: a NaN or both sides of the iso value in
    the block's dilated window), the fine pass evaluates the 729 points of each active block, and marching cubes runs
    over those blocks.  The result is extract_mesh's mesh without the triangles of inactive blocks (and the vertices
    only they used); it equals extract_mesh's whenever every cell the surface crosses is in an active block.  A feature
    smaller than a block that no coarse point sees can be missed.  opt.trimesh.res must be a multiple of 8 (ValueError
    otherwise).  stats: an optional dict that receives n_blocks, n_active and points_evaluated."""
    res, rng, thres = trimesh_settings(opt)
    check_sparse_res(res)
    axis = lattice_axis(res, rng)
    slots, block_ids = ops.mcubes_sparse_classify(coarse_density(nerf, axis, engine=engine), thres)
    sigma = block_density(nerf, axis, block_ids, engine=engine)
    verts, faces = ops.marching_cubes_sparse(sigma, res, slots, block_ids, thres)
    if stats is not None:
        nb = res // BLOCK
        stats.update(n_blocks=nb ** 3, n_active=block_ids.numel(),
                     points_evaluated=(nb + 1) ** 3 + block_ids.numel() * (BLOCK + 1) ** 3)
    del sigma
    out = dict(vertices=to_world(verts, res, rng), faces=faces)
    if normals:
        out["normals"] = density_normals(nerf, out["vertices"], engine=engine)
    return out


def write_ply(path, vertices, faces, normals=None, colors=None) -> None:
    """Binary little-endian PLY: float x, y, z (and nx, ny, nz) per vertex, then, when colors [V, 3] is given, uchar
    red, green, blue = round(clamp(c, 0, 1) * 255) (to nearest, ties to even); a uchar-counted int list per face"""
    as_np = lambda x: x.detach().cpu().numpy() if torch.is_tensor(x) else np.asarray(x)
    v = as_np(vertices).astype(np.float32).reshape(-1, 3)
    f = as_np(faces).astype(np.int64).reshape(-1, 3)
    assert f.size == 0 or (f.min() >= 0 and f.max() < min(len(v), 2 ** 31)), "face ids out of range"
    names = ["x", "y", "z"] + (["nx", "ny", "nz"] if normals is not None else [])
    rgb = ["red", "green", "blue"] if colors is not None else []
    vert = np.empty(len(v), np.dtype([(k, "<f4") for k in names] + [(k, "u1") for k in rgb]))
    for c, k in enumerate("xyz"):
        vert[k] = v[:, c]
    if normals is not None:
        nrm = as_np(normals).astype(np.float32).reshape(-1, 3)
        assert len(nrm) == len(v)
        for c, k in enumerate(["nx", "ny", "nz"]):
            vert[k] = nrm[:, c]
    if colors is not None:
        col = as_np(colors).astype(np.float32).reshape(-1, 3)
        assert len(col) == len(v)
        col = np.round(np.clip(col, 0.0, 1.0) * np.float32(255)).astype(np.uint8)
        for c, k in enumerate(rgb):
            vert[k] = col[:, c]
    face = np.empty(len(f), np.dtype([("n", "u1"), ("v", "<i4", (3,))]))
    face["n"] = 3
    face["v"] = f
    header = ["ply", "format binary_little_endian 1.0", "element vertex %d" % len(v)]
    header += ["property float %s" % k for k in names] + ["property uchar %s" % k for k in rgb]
    header += ["element face %d" % len(f), "property list uchar int vertex_indices", "end_header"]
    with open(path, "wb") as fh:
        fh.write(("\n".join(header) + "\n").encode("ascii"))
        fh.write(vert.tobytes())
        fh.write(face.tobytes())
