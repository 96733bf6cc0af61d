"""Mesh extraction from a trained NeRF, BARF's recipe on the device: the density on the lattice of `opt.trimesh`
(train_settings/default_config.py:267-271), marching cubes (csrc/mcubes.cu), world coordinates, optional normals from
the density's gradient, floater removal by connected components (keep_components), simplification (simplify),
measurement against a reference surface (compare: Chamfer distance, F-score), ray casting (render: mesh depth maps;
visible_faces and cull: the part of a mesh that cameras see), and a PLY writer and reader.

    from sparf_b200 import mesh
    m = mesh.extract_mesh(opt, graph.nerf, normals=True)        # or graph.nerf_fine
    m = mesh.keep_components(m, largest=1)                      # optional: drop the floaters
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


VERTEX_KEYS = ("vertices", "normals", "colors")     # the per-vertex entries of the extractors' mesh dicts


def keep_components(m: dict, largest=None, min_faces: int = 1, stats=None) -> dict:
    """Floater removal for a mesh dict of extract_mesh, extract_mesh_sparse or tsdf.extract_mesh: the connected
    components (ops.mesh_components; two vertices are connected when a face holds both) with at least min_faces faces,
    and of those, when largest = k, only the k largest by (face count descending, label ascending).  -> a dict with the
    same keys: the kept faces in their order with renumbered ids, and the kept vertices in their order with their
    vertices / normals / colors gathered (ops.mesh_select), ready for write_ply.  Other entries are passed on as they
    are.  stats: an optional dict that receives n_components, n_kept (components kept) and faces_removed."""
    if largest is not None and (isinstance(largest, bool) or not isinstance(largest, int) or largest < 1):
        raise ValueError("keep_components: largest must be None or an int >= 1 (got %r)" % (largest,))
    if isinstance(min_faces, bool) or not isinstance(min_faces, int) or min_faces < 0:
        raise ValueError("keep_components: min_faces must be an int >= 0 (got %r)" % (min_faces,))
    faces, n_verts = m["faces"], m["vertices"].shape[0]
    labels, counts = ops.mesh_components(faces, n_verts)
    kept = torch.nonzero(counts >= min_faces).flatten()         # increasing labels
    if largest is not None:
        order = torch.sort(counts[kept], descending=True, stable=True).indices   # ties: the smaller label first
        kept = kept[order[:largest]]
    keep = torch.zeros(counts.numel(), dtype=torch.uint8, device=counts.device)
    keep[kept] = 1
    vert_ids, faces_out = ops.mesh_select(faces, n_verts, labels, keep)
    out = dict(m)
    out["faces"] = faces_out
    for k in VERTEX_KEYS:
        if m.get(k) is not None:
            out[k] = m[k][vert_ids]
    if stats is not None:
        stats.update(n_components=counts.numel(), n_kept=kept.numel(), faces_removed=faces.shape[0] - faces_out.shape[0])
    return out


def simplify(m: dict, target_faces: int, stats=None) -> dict:
    """Quadric-error simplification (ops.mesh_simplify) of a mesh dict of extract_mesh, extract_mesh_sparse or
    tsdf.extract_mesh, before or after keep_components, to at most target_faces faces where the edge collapses reach
    it.  Boundary and non-manifold vertices stay where they are.  normals and colors are interpolated along the
    collapses; the normals are then made unit again by unit_normals' rule (0 where the length is 0).  Other entries are
    passed on as they are.  stats: an optional dict that receives rounds, collapses, faces_before, faces_after and
    reached (faces_after <= target_faces)."""
    keys = [k for k in VERTEX_KEYS[1:] if m.get(k) is not None]
    attrs = torch.cat([m[k] for k in keys], dim=1) if keys else None
    st = {}
    verts, faces, _, attrs = ops.mesh_simplify(m["vertices"], m["faces"], target_faces, attrs=attrs, stats=st)
    out = dict(m, vertices=verts, faces=faces)
    col = 0
    for k in keys:
        out[k] = attrs[:, col:col + m[k].shape[1]]
        col += m[k].shape[1]
    if "normals" in keys:
        out["normals"] = unit_normals(-out["normals"])
    if stats is not None:
        stats.update(st, faces_before=m["faces"].shape[0], faces_after=faces.shape[0],
                     reached=faces.shape[0] <= target_faces)
    return out


def sample_surface(m: dict, n: int, seed: int = 0) -> torch.Tensor:
    """n points [n, 3] (fp32) on the triangles of the mesh dict m, uniform over its area: a face by searchsorted of fp64
    uniforms (scaled to the total) in the fp64 cumulative face areas, a point in it at the barycentrics (1 - sqrt(u1),
    sqrt(u1) (1 - u2), sqrt(u1) u2).  The uniforms come from a torch.Generator on the mesh's device seeded with seed.
    A mesh without faces or area gives no points."""
    if isinstance(n, bool) or not isinstance(n, int) or n < 0:
        raise ValueError("sample_surface: n must be an int >= 0 (got %r)" % (n,))
    v, f = m["vertices"], m["faces"]
    dev = v.device
    p = v.double()[f] if f.numel() else torch.zeros(0, 3, 3, dtype=torch.float64, device=dev)
    area = torch.linalg.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0]).norm(dim=1) / 2
    cum = torch.cumsum(area, 0)
    if n == 0 or cum.numel() == 0 or not cum[-1].item() > 0:
        return torch.zeros(0, 3, dtype=torch.float32, device=dev)
    g = torch.Generator(device=dev)
    g.manual_seed(seed)
    u = torch.rand(3, n, generator=g, device=dev, dtype=torch.float64)
    face = torch.searchsorted(cum, u[0] * cum[-1], right=True).clamp_(max=cum.numel() - 1)
    s = u[1].sqrt()
    w = torch.stack([1 - s, s * (1 - u[2]), s * u[2]], 1)
    return (w[:, :, None] * p[face]).sum(1).float()


def distance_metrics(d_acc: torch.Tensor, d_comp: torch.Tensor, threshold: float, max_dist=float("inf")) -> dict:
    """The metrics of compare from the distances of the pred samples to ref (d_acc) and of the ref samples to pred
    (d_comp), misses as inf: accuracy / completeness = the fp64 means of min(d, max_dist) (NaN over no samples),
    chamfer = their mean, precision / recall = the fractions with d < threshold (0 over no samples), fscore = 2PR /
    (P + R) (0 when P + R = 0), hausdorff = the larger maximum of min(d, max_dist) (of the sides with samples; NaN
    when neither has any), n_pred, n_ref."""
    out = dict(n_pred=int(d_acc.numel()), n_ref=int(d_comp.numel()))
    means, fracs, maxes = [], [], []
    for d in (d_acc, d_comp):
        d = d.double().clamp(max=float(max_dist))
        means.append(d.mean().item() if d.numel() else float("nan"))
        fracs.append((d < threshold).double().mean().item() if d.numel() else 0.0)
        if d.numel():
            maxes.append(d.max().item())
    P, R = fracs
    out.update(accuracy=means[0], completeness=means[1], chamfer=(means[0] + means[1]) / 2, precision=P, recall=R,
               fscore=2 * P * R / (P + R) if P + R > 0 else 0.0, hausdorff=max(maxes) if maxes else float("nan"))
    return out


def _phase(phases, name, fn):
    """fn(), its synchronised wall time added to phases[name] (s) when phases is a dict"""
    if phases is None:
        return fn()
    import time
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    phases[name] = phases.get(name, 0.0) + time.perf_counter() - t
    return out


def prepare(m: dict, n_samples: int = 1_000_000, seed: int = 0, stats=None) -> dict:
    """One side of compare, ready to be compared many times: m with "points" (n_samples surface samples of a mesh,
    sample_surface with seed; the vertices of a point cloud, a dict without faces) and "grid" (ops.distance_grid of its
    triangles, or of its points).  A dict that already has both is returned as it is.  stats: an optional dict that
    receives the time of the sample and grid phases (s)."""
    if m.get("grid") is not None and m.get("points") is not None:
        return m
    if m.get("faces") is not None:
        pts = _phase(stats, "sample", lambda: sample_surface(m, n_samples, seed))
        grid = _phase(stats, "grid", lambda: ops.distance_grid(m["vertices"], m["faces"]))
    else:
        pts = m["vertices"]
        grid = _phase(stats, "grid", lambda: ops.distance_grid(m["vertices"]))
    return dict(m, points=pts, grid=grid)


def compare(pred: dict, ref: dict, threshold: float, n_samples: int = 1_000_000, max_dist=float("inf"), seed: int = 0,
            stats=None) -> dict:
    """How close the mesh dict pred is to the reference ref (a mesh dict, or a point cloud: a dict without faces, such as
    DTU's reference scans): accuracy = the mean distance of pred's samples to ref, completeness = of ref's samples to
    pred, chamfer = their mean; precision, recall and their fscore at threshold; hausdorff; n_pred, n_ref
    (distance_metrics).  A side with faces is sampled with n_samples points (sample_surface, seeds seed for pred and
    seed + 1 for ref), a point cloud is used as it is; each side's primitives are its triangles, or its points.  The
    distances are exact (ops.closest_points), capped at max_dist.  Either side may be a prepare()d dict, so that
    scoring several meshes against one reference samples it and builds its grid once.  Masks and crops are the
    caller's: filter the points before the call.  stats: an optional dict that receives the time of the sample, grid
    and query phases (s, synchronised)."""
    if not threshold > 0:
        raise ValueError("compare: threshold must be > 0 (got %r)" % (threshold,))
    if not max_dist >= 0:
        raise ValueError("compare: max_dist must be >= 0 or inf (got %r)" % (max_dist,))
    pred = prepare(pred, n_samples, seed, stats)
    ref = prepare(ref, n_samples, seed + 1, stats)
    d_acc = _phase(stats, "query", lambda: ops.closest_points(ref["grid"], pred["points"], max_dist)[0])
    d_comp = _phase(stats, "query", lambda: ops.closest_points(pred["grid"], ref["points"], max_dist)[0])
    return distance_metrics(d_acc, d_comp, threshold, max_dist)


def _check_views(m, pose_w2c, intr, H, W, masks, grid, what, near=0.0, far=float("inf")):
    """(B, the ray-cast grid or None when it is to be built) after ValueError checks that need no library call"""
    real = lambda x: isinstance(x, (int, float)) and not isinstance(x, bool)
    if not real(near) or not real(far) or not 0 <= near <= far:
        raise ValueError("%s: need 0 <= near <= far (inf allowed), got %r, %r" % (what, near, far))
    if not isinstance(m, dict) or not torch.is_tensor(m.get("vertices")) or not torch.is_tensor(m.get("faces")):
        raise ValueError("%s: m must be a mesh dict with vertices and faces" % what)
    if not torch.is_tensor(pose_w2c) or pose_w2c.dtype != torch.float32 or pose_w2c.dim() != 3 \
            or tuple(pose_w2c.shape[1:]) != (3, 4) or pose_w2c.shape[0] < 1:
        raise ValueError("%s: pose_w2c must be a float32 tensor [B, 3, 4] with B >= 1" % what)
    B = pose_w2c.shape[0]
    if not torch.is_tensor(intr) or intr.dtype != torch.float32 or tuple(intr.shape) not in ((3, 3), (B, 3, 3)):
        raise ValueError("%s: intr must be a float32 tensor [3, 3] or [%d, 3, 3]" % (what, B))
    for name, n in (("H", H), ("W", W)):
        if isinstance(n, bool) or not isinstance(n, int) or n < 1:
            raise ValueError("%s: %s must be an int >= 1 (got %r)" % (what, name, n))
    if masks is not None and (not torch.is_tensor(masks) or masks.dtype not in (torch.bool, torch.uint8)
                              or tuple(masks.shape) != (B, H, W)):
        raise ValueError("%s: masks must be None or a bool / uint8 tensor [%d, %d, %d]" % (what, B, H, W))
    dev = m["vertices"].device
    if dev.type != "cuda" or any(x is not None and x.device != dev for x in (m["faces"], pose_w2c, intr, masks)):
        raise ValueError("%s: the mesh, cameras and masks must be on one CUDA device" % what)
    grid = grid if grid is not None else m.get("grid")
    if grid is not None and (not isinstance(grid, ops.DistanceGrid) or grid.faces is None):
        raise ValueError("%s: grid must be an ops.DistanceGrid of the mesh's triangles" % what)
    return B, grid


def _cast_views(m, pose_w2c, intr, H, W, near, far, grid):
    """ops.raycast of the pixel-centre rays of every view (camera.get_center_and_ray) in chunks of about
    tsdf.BATCH_PIXELS rays: yields (b0, b1, p0, p1, t, face, bary), the results for views b0..b1-1 and pixels p0..p1-1
    as [b1 - b0, p1 - p0] (bary [..., 3])"""
    from . import camera, tsdf
    grid = grid if grid is not None else ops.distance_grid(m["vertices"], m["faces"])
    B, HW = pose_w2c.shape[0], H * W
    intr = intr.expand(B, 3, 3) if intr.dim() == 2 else intr
    per_view = max(1, tsdf.BATCH_PIXELS // HW)
    pix = min(HW, tsdf.BATCH_PIXELS)
    for b0 in range(0, B, per_view):
        b1 = min(B, b0 + per_view)
        for p0 in range(0, HW, pix):
            p1 = min(HW, p0 + pix)
            idx = torch.arange(p0, p1, device=pose_w2c.device)
            o, d = camera.get_center_and_ray(pose_w2c[b0:b1], H, W, intr[b0:b1], ray_idx=idx)
            t, face, bary = ops.raycast(grid, o.reshape(-1, 3), d.reshape(-1, 3), near, far)
            n = p1 - p0
            yield b0, b1, p0, p1, t.view(-1, n), face.view(-1, n), bary.view(-1, n, 3)


@torch.no_grad()
def render(m: dict, pose_w2c, intr, H: int, W: int, near: float = 0.0, far: float = float("inf"), grid=None) -> dict:
    """Depth maps of the mesh dict m from B views, pose_w2c [B, 3, 4] and intr [B, 3, 3] or [3, 3] (fp32, on the
    mesh's CUDA device), H x W pixels: the first hit (ops.raycast, t in [near, far]) of each pixel-centre ray of
    camera.get_center_and_ray.  -> dict(depth [B, H, W] fp32: t, the camera z-depth as in tsdf.render_maps, inf at
    misses; face [B, H, W] int64, -1 at misses; bary [B, H, W, 3] fp32, NaN at misses), plus for each per-vertex entry
    of m (normals, colors) its barycentric interpolation at the hit [B, H, W, C], NaN at misses.  The grid is grid if
    given, else m["grid"] of a prepare()d dict, else ops.distance_grid of m's triangles.  ValueError for bad arguments
    before any library call."""
    B, grid = _check_views(m, pose_w2c, intr, H, W, None, grid, "render", near, far)
    dev = m["vertices"].device
    out = dict(depth=torch.empty(B, H * W, device=dev), face=torch.empty(B, H * W, dtype=torch.int64, device=dev),
               bary=torch.empty(B, H * W, 3, device=dev))
    for b0, b1, p0, p1, t, face, bary in _cast_views(m, pose_w2c, intr, H, W, near, far, grid):
        out["depth"][b0:b1, p0:p1] = t
        out["face"][b0:b1, p0:p1] = face
        out["bary"][b0:b1, p0:p1] = bary
    f = m["faces"]
    for k in VERTEX_KEYS[1:]:
        if m.get(k) is None:
            continue
        a = m[k]
        if f.shape[0] == 0:
            out[k] = torch.full((B, H * W, a.shape[1]), float("nan"), device=dev)
            continue
        corners = a[f[out["face"].clamp(min=0)]]                       # [B, HW, 3, C]
        out[k] = (out["bary"][..., None] * corners).sum(-2)            # NaN barycentrics at misses give NaN
    for k, v in out.items():
        out[k] = v.view(B, H, W, *v.shape[2:])
    return out


@torch.no_grad()
def visible_faces(m: dict, pose_w2c, intr, H: int, W: int, masks=None, grid=None) -> torch.Tensor:
    """bool [F]: the faces of the mesh dict m that are the first hit (render's) of the pixel-centre ray of at least one
    pixel of at least one view, counting only the pixels inside masks [B, H, W] (bool / uint8) when given.  Visibility
    is sampled at pixel centres, as a rasterizer samples coverage: a face that no pixel centre hits first (smaller than
    a pixel, or seen only edge-on) is not visible."""
    B, grid = _check_views(m, pose_w2c, intr, H, W, masks, grid, "visible_faces")
    F = m["faces"].shape[0]
    vis = torch.zeros(F, dtype=torch.bool, device=m["vertices"].device)
    flat = masks.reshape(B, H * W) if masks is not None else None
    for b0, b1, p0, p1, _, face, _ in _cast_views(m, pose_w2c, intr, H, W, 0.0, float("inf"), grid):
        keep = face >= 0
        if flat is not None:
            keep &= flat[b0:b1, p0:p1].bool()
        vis[face[keep]] = True
    return vis


@torch.no_grad()
def cull(m: dict, pose_w2c, intr, H: int, W: int, masks=None, stats=None) -> dict:
    """The part of the mesh dict m that the views see (visible_faces, with masks [B, H, W] when given): the visible
    faces in their order with renumbered ids, and the vertices they use in their order with their vertices / normals /
    colors gathered; other entries are passed on as they are (the output of keep_components, so cull, keep_components,
    simplify and compare chain), except the points and grid of a prepare()d dict, which describe the uncut mesh and are
    dropped.  DTU's evaluation culls a predicted mesh this way before scoring it.  stats: an optional dict that receives
    faces_before, faces_after, views and pixels (the rays cast)."""
    B, _ = _check_views(m, pose_w2c, intr, H, W, masks, None, "cull")
    faces = m["faces"]
    vis = visible_faces(m, pose_w2c, intr, H, W, masks=masks)
    kept = faces[vis]
    used = torch.zeros(m["vertices"].shape[0], dtype=torch.bool, device=faces.device)
    used[kept.reshape(-1)] = True
    new_id = torch.cumsum(used, 0) - 1
    out = {k: v for k, v in m.items() if k not in ("points", "grid")}
    out["faces"] = new_id[kept]
    vert_ids = torch.nonzero(used).flatten()
    for k in VERTEX_KEYS:
        if m.get(k) is not None:
            out[k] = m[k][vert_ids]
    if stats is not None:
        stats.update(faces_before=faces.shape[0], faces_after=kept.shape[0], views=B, pixels=B * H * W)
    return out


_PLY_TYPES = {"char": "i1", "int8": "i1", "uchar": "u1", "uint8": "u1", "short": "i2", "int16": "i2", "ushort": "u2",
              "uint16": "u2", "int": "i4", "int32": "i4", "uint": "u4", "uint32": "u4", "float": "f4", "float32": "f4",
              "double": "f8", "float64": "f8"}


def read_ply(path) -> dict:
    """A PLY file (ascii or binary_little_endian) as a mesh dict: vertices [V, 3] fp32 from x, y, z; normals from nx,
    ny, nz and colors (fp32; uchar / 255) from red, green, blue when present; faces [F, 3] int64 from the vertex_indices
    (or vertex_index) list of the face element, or no faces entry when the file has no face element (a point cloud).
    Any scalar type; other vertex properties are skipped.  Big-endian files, faces that are not triangles and list
    properties other than the face list in a binary file raise ValueError.  The tensors are on the CPU."""
    with open(path, "rb") as fh:
        data = fh.read()
    end = data.find(b"end_header")
    if not data.startswith(b"ply") or end < 0:
        raise ValueError("read_ply: %s is not a PLY file" % path)
    body = data.index(b"\n", end) + 1
    fmt, elements = None, []
    for line in data[:end].decode("ascii", "replace").splitlines()[1:]:
        w = line.split()
        if not w or w[0] in ("comment", "obj_info"):
            continue
        if w[0] == "format":
            fmt = w[1]
        elif w[0] == "element":
            elements.append((w[1], int(w[2]), []))
        elif w[0] == "property" and elements:
            if w[1] == "list":
                if w[2] not in _PLY_TYPES or w[3] not in _PLY_TYPES:
                    raise ValueError("read_ply: unknown list type in %r" % line)
                elements[-1][2].append((w[4], (_PLY_TYPES[w[2]], _PLY_TYPES[w[3]])))
            else:
                if w[1] not in _PLY_TYPES:
                    raise ValueError("read_ply: unknown property type in %r" % line)
                elements[-1][2].append((w[2], _PLY_TYPES[w[1]]))
    if fmt not in ("ascii", "binary_little_endian"):
        raise ValueError("read_ply: format %r is not supported (ascii or binary_little_endian)" % fmt)
    arrays = _ply_ascii(data[body:], elements) if fmt == "ascii" else _ply_binary(data[body:], elements)
    vert = arrays.get("vertex")
    if vert is None or not all(k in vert for k in "xyz"):
        raise ValueError("read_ply: %s has no vertex element with x, y, z" % path)
    cols = lambda names: np.stack([np.asarray(vert[k], np.float64) for k in names], 1)
    out = dict(vertices=torch.from_numpy(cols("xyz").astype(np.float32)).reshape(-1, 3))
    if all(k in vert for k in ("nx", "ny", "nz")):
        out["normals"] = torch.from_numpy(cols(["nx", "ny", "nz"]).astype(np.float32)).reshape(-1, 3)
    if all(k in vert for k in ("red", "green", "blue")):
        c = cols(["red", "green", "blue"])
        if vert["red"].dtype == np.uint8:
            c = c / 255.0
        out["colors"] = torch.from_numpy(c.astype(np.float32)).reshape(-1, 3)
    if "face" in arrays:
        out["faces"] = torch.from_numpy(arrays["face"]).reshape(-1, 3)
    return out


def _face_list(props):
    names = [n for n, _ in props]
    for key in ("vertex_indices", "vertex_index"):
        if key in names:
            return key
    return None


def _ply_ascii(text, elements):
    words = text.split()
    pos, out = 0, {}
    for name, count, props in elements:
        if name == "face" and count and _face_list(props) is None:
            raise ValueError("read_ply: the face element has no vertex_indices list")
        cols = {n: [] for n, _ in props}
        faces = []
        for _ in range(count):
            for n, t in props:
                if isinstance(t, tuple):
                    k = int(words[pos])
                    vals = [int(x) for x in words[pos + 1:pos + 1 + k]]
                    pos += 1 + k
                    if name == "face" and n == _face_list(props):
                        if k != 3:
                            raise ValueError("read_ply: a face with %d vertices (only triangles)" % k)
                        faces.append(vals)
                else:
                    cols[n].append(float(words[pos]))
                    pos += 1
        if name == "vertex":
            out["vertex"] = {n: np.asarray(cols[n], np.float64).astype(t) for n, t in props if not isinstance(t, tuple)}
        elif name == "face":
            out["face"] = np.asarray(faces, np.int64).reshape(-1, 3)
    return out


def _ply_binary(buf, elements):
    pos, out = 0, {}
    for name, count, props in elements:
        lists = [(n, t) for n, t in props if isinstance(t, tuple)]
        if not lists:
            dt = np.dtype([(n, "<" + t) for n, t in props])
            arr = np.frombuffer(buf, dt, count, pos)
            pos += dt.itemsize * count
            if name == "vertex":
                out["vertex"] = {n: arr[n] for n, _ in props}
            continue
        if name != "face" or len(props) != 1 or _face_list(props) is None:
            raise ValueError("read_ply: binary list properties are only read as the face element's vertex list")
        ct, it = np.dtype("<" + props[0][1][0]), np.dtype("<" + props[0][1][1])
        if count:
            k = int(np.frombuffer(buf, ct, 1, pos)[0])
            if k != 3:
                raise ValueError("read_ply: a face with %d vertices (only triangles)" % k)
            rec = np.dtype([("n", ct), ("v", it, (3,))])
            arr = np.frombuffer(buf, rec, count, pos)
            if (arr["n"] != 3).any():
                raise ValueError("read_ply: a face that is not a triangle")
            pos += rec.itemsize * count
            out["face"] = arr["v"].astype(np.int64)
        else:
            out["face"] = np.zeros((0, 3), np.int64)
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
