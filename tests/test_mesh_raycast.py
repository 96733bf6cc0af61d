"""GPU tests of the mesh ray cast (csrc/mesh_raycast.cu, ops.raycast, mesh.render / visible_faces / cull): agreement
with the fp64 oracle (tests/raycast_oracle.py) on the meshes of test_mesh_distance.py; identical bytes for every grid,
also for rays built from the grid's own planes; watertightness on closed meshes; analytic depth maps; culling; the
project's extractors; CUDA-graph capture; empty cases; a 6 M-face mesh against three DTU-sized views; and the tools."""
import math
import os
import sys

import numpy as np
import pytest
import torch

import raycast_oracle as RO
import mesh_distance_oracle as MD
import test_mesh_components as TMC
import test_mesh_distance as TMD

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ULP = 2.0 ** -24
MESHES = TMD.MESHES


def _bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def _same(a, b):
    return all(torch.equal(_bits(x), _bits(y)) for x, y in zip(a, b))


def _unit(x):
    return x / x.norm(dim=1, keepdim=True)


def _normals(v, f):
    a, b, c = (v[f[:, k]] for k in range(3))
    return torch.linalg.cross(b - a, c - a)


def _rays(v, f, seed=0):
    """{kind: (origins, dirs, t_min)}: from outside the box at the surface, from inside the box, from the surface
    (t_min > 0), grazing and parallel to faces, with zero direction components, and NaN / zero-length rays"""
    from sparf_b200 import mesh
    g = torch.Generator(device="cuda").manual_seed(seed)
    lo, hi = v.min(0).values, v.max(0).values
    c, ext = (lo + hi) / 2, (hi - lo).max().item()
    on = mesh.sample_surface(dict(vertices=v, faces=f), 600, seed=seed)
    n = len(on)
    far = c + 1.5 * ext * _unit(torch.randn(n, 3, generator=g, device="cuda"))
    out = dict(outside=(far, on + 0.05 * ext * torch.randn(n, 3, generator=g, device="cuda") - far, 0.0))
    inside = lo + (hi - lo) * torch.rand(n, 3, generator=g, device="cuda")
    out["inside"] = (inside, torch.randn(n, 3, generator=g, device="cuda"), 0.0)
    out["surface"] = (on, torch.randn(n, 3, generator=g, device="cuda"), 1e-3 * ext)
    # tangent to the face under a surface point: grazing it, and parallel to it just above
    from sparf_b200 import ops
    _, idx, _ = ops.closest_points(ops.distance_grid(v, f), on)
    nrm = _normals(v, f)[idx]
    tang = _unit(torch.linalg.cross(nrm, torch.randn(n, 3, generator=g, device="cuda")))
    out["grazing"] = (on - 0.7 * ext * tang, tang, 0.0)
    out["parallel"] = (on - 0.7 * ext * tang + 1e-3 * ext * _unit(nrm), tang, 0.0)
    d = torch.randn(n, 3, generator=g, device="cuda")
    d[: n // 3, 0] = 0
    d[n // 3: 2 * n // 3, 1:] = 0
    out["axes"] = (inside, d, 0.0)
    bad_o = inside[:8].clone()
    bad_d = torch.randn(8, 3, generator=g, device="cuda")
    bad_o[0, 1] = float("nan")
    bad_d[1, 2] = float("nan")
    bad_d[2:4] = 0
    bad_d[4, 0] = float("inf")
    out["bad"] = (bad_o, bad_d, 0.0)
    return out


def _bound(o, v):
    """the agreement bound in coordinates: 64 ulps of |o|_inf + the mesh's largest |coordinate|"""
    return 64 * ULP * (np.abs(o).max(1) + np.abs(v).max())


def _near_boundary(p, vn, fn, ids, b):
    """the points p [N, 3] that lie within b of an edge of triangle ids"""
    tri = vn[fn[ids]]
    d = np.full(len(p), np.inf)
    for i, j in ((0, 1), (1, 2), (2, 0)):
        q = MD.closest_on_segment(p, tri[:, i], tri[:, j])
        d = np.minimum(d, np.linalg.norm(p - q, axis=1))
    return d <= b


def _check_against_oracle(v, f, o, d, t_min=0.0, t_max=float("inf"), grid=None):
    """misses exactly inf / -1 / NaN; a hit lies on its face and realises t (within the bound), its barycentrics
    reproduce the hit point, and (t, face) is the oracle's unless the two disagree only at a triangle's edge or at a
    t within the bound; an oracle hit the kernel misses lies at an edge (a silhouette)"""
    from sparf_b200 import ops
    grid = grid or ops.distance_grid(v, f)
    t, face, bary = (x.cpu().numpy() for x in ops.raycast(grid, o, d, t_min, t_max))
    vn, fn = v.cpu().numpy().astype(np.float64), f.cpu().numpy()
    on, dn = o.cpu().numpy().astype(np.float64), d.cpu().numpy().astype(np.float64)
    t64, f64, _ = RO.raycast(on, dn, vn, fn, t_min, t_max)
    b = _bound(on, vn)
    dl = np.linalg.norm(dn, axis=1)
    with np.errstate(invalid="ignore"):
        bt = b / np.where(dl > 0, dl, np.nan)
    miss = face < 0
    assert np.isinf(t[miss]).all() and (t[miss] > 0).all() and np.isnan(bary[miss]).all()
    h = ~miss
    assert ((t[h] >= t_min) & (t[h] <= t_max)).all()

    def cond_of(ids, m):
        """1 + 1 / cos^2 of the incidence of rays m on faces ids: a rounding error of b across the plane moves a hit by
        up to b times that along the ray"""
        tri = vn[fn[ids]]
        n = np.cross(tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0])
        cos = np.abs((n * dn[m]).sum(1)) / (np.linalg.norm(n, axis=1) * dl[m])
        return 1 + 1 / np.maximum(cos, 1e-30) ** 2

    cond = np.ones(len(t))
    cond[h] = cond_of(face[h], h)
    p = on[h] + t[h, None].astype(np.float64) * dn[h]
    on_tri, _ = MD.triangle_distance(p, vn, fn, face[h])
    assert (on_tri <= b[h] * cond[h]).all(), np.max(on_tri / (b[h] * cond[h]))
    pb = (bary[h, :, None].astype(np.float64) * vn[fn[face[h]]]).sum(1)
    assert (np.linalg.norm(pb - p, axis=1) <= b[h] * cond[h]).all()
    assert (np.abs(bary[h].sum(1) - 1) <= 1e-5).all() and (bary[h] >= 0).all()
    at_bounds = lambda tt, m: (np.abs(tt - t_min) <= bt[m] * cond[m]) | (np.abs(tt - t_max) <= bt[m] * cond[m])

    def at_edge(tt, ids, m):
        """the hits at tt on faces ids of rays m that lie at an edge of their face, within the hit's conditioning"""
        pt = on[m] + tt[:, None].astype(np.float64) * dn[m]
        return _near_boundary(pt, vn, fn, ids, b[m] * cond_of(ids, m))

    # the kernel missed an oracle hit: only at an edge, or at t_min / t_max
    lost = miss & (f64 >= 0)
    if lost.any():
        assert (at_edge(t64[lost], f64[lost], lost) | at_bounds(t64[lost], lost)).all()
    # both hit: the same face, or t within the bound, or one of the two hits at an edge or at t_min / t_max
    both = h & (f64 >= 0)
    diff = both & (face != f64)
    if diff.any():
        ok = np.abs(t[diff] - t64[diff]) <= bt[diff]
        ok |= at_edge(t[diff], face[diff], diff) | at_bounds(t[diff], diff)
        ok |= at_edge(t64[diff], f64[diff], diff) | at_bounds(t64[diff], diff)
        assert ok.all()
    # the kernel hit where the oracle missed: at an edge or at t_min / t_max
    extra = h & (f64 < 0)
    if extra.any():
        assert (at_edge(t[extra], face[extra], extra) | at_bounds(t[extra], extra)).all()
    # t of the same face: within the bound scaled by the hit's conditioning (1 + 1 / cos^2 of the incidence)
    same = both & (face == f64)
    assert (np.abs(t[same] - t64[same]) <= bt[same] * cond[same]).all()
    return t, face, bary


# ------------------------------------------------------------------------------------------------ 1. oracle agreement
@pytest.mark.parametrize("name", sorted(MESHES))
def test_matches_oracle(name):
    v, f = MESHES[name]()
    for kind, (o, d, t_min) in _rays(v, f).items():
        t, face, _ = _check_against_oracle(v, f, o, d, t_min)
        if kind == "bad":
            assert (face[:5] == -1).all() and np.isinf(t[:5]).all()
        ext = (v.max(0).values - v.min(0).values).max().item()
        _check_against_oracle(v, f, o, d, t_min, t_max=0.5 * ext)


# ------------------------------------------------------------------------------------------------ 2. exactness
def _plane_rays(grid, n=400, seed=0):
    """rays built from the grid's planes: through cell corners, along cell edges and faces, axis-aligned rays lying in a
    cell plane"""
    lo = grid.params[:12].view(torch.float32)[:3].double()
    cell = grid.params[12:24].view(torch.float32).double()
    dims = torch.tensor(grid.dims, device="cuda")
    g = torch.Generator(device="cuda").manual_seed(seed)
    corner = lambda: lo + cell * torch.stack([torch.randint(0, int(m) + 1, (n,), generator=g, device="cuda")
                                              for m in dims], 1).double()
    a, b = corner(), corner()
    o, d = [a.float()], [(b - a).float()]                          # corner to corner
    e = torch.zeros(n, 3, dtype=torch.float64, device="cuda")
    ax = torch.randint(0, 3, (n,), generator=g, device="cuda")
    e[torch.arange(n), ax] = 1.0
    o.append((a - 2 * e * cell * dims).float())
    d.append(e.float())                                             # along cell edges, axis-aligned
    w = torch.randn(n, 3, generator=g, device="cuda", dtype=torch.float64)
    w[torch.arange(n), ax] = 0
    o.append(a.float())
    d.append(w.float())                                             # in a cell plane
    o.append((a + 0.5 * cell * e).float())
    d.append((w + 0.3 * e).float())                                 # across planes from mid-cell
    return torch.cat(o).contiguous(), torch.cat(d).contiguous()


@pytest.mark.parametrize("name", sorted(MESHES))
def test_same_bytes_for_every_grid(name):
    from sparf_b200 import ops
    v, f = MESHES[name]()
    rays = list(_rays(v, f, seed=4).values())
    default = ops.distance_grid(v, f)
    o = torch.cat([r[0] for r in rays] + [_plane_rays(default)[0], _plane_rays(ops.distance_grid(v, f, 17))[0]])
    d = torch.cat([r[1] for r in rays] + [_plane_rays(default)[1], _plane_rays(ops.distance_grid(v, f, 17))[1]])
    ref = ops.raycast(default, o, d)
    assert (ref[1] >= 0).sum() > 100
    for c in [1, 3, 17, None, tuple(4 * x for x in default.dims)]:
        g = ops.distance_grid(v, f, cells_per_axis=c)
        for _ in range(2):
            assert _same(ops.raycast(g, o, d), ref), c
            assert _same(ops.raycast(g, o, d, 0.1, 30.0), ops.raycast(default, o, d, 0.1, 30.0)), c
    _check_against_oracle(v, f, o, d)


# ------------------------------------------------------------------------------------------------ 3. watertight
@pytest.mark.parametrize("name", ["sphere", "torus"])
def test_closed_meshes_are_watertight(name):
    """every ray from an interior point hits, also rays aimed exactly at vertices and at edge midpoints"""
    from sparf_b200 import ops
    v, f = TMD._sphere(30, 11.0) if name == "sphere" else TMD._torus(40, 11.0, 5.0)
    c = (30 - 1) / 2 + 0.13 if name == "sphere" else (40 - 1) / 2 + 0.11
    if name == "sphere":
        inner = torch.tensor([[c, c, c], [c + 3.1, c - 2.2, c + 1.7]], device="cuda")
    else:      # on the tube's centre circle (the torus lies around axis 2)
        a = torch.tensor([0.3, 2.1, 4.4], device="cuda")
        inner = torch.stack([c + 11.0 * torch.cos(a), c + 11.0 * torch.sin(a), torch.full_like(a, c)], 1)
    e = torch.cat([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
    targets = torch.cat([v, (v[e[:, 0]] + v[e[:, 1]]) / 2])
    grid = ops.distance_grid(v, f)
    for p in inner:
        o = p.expand_as(targets).contiguous()
        t, face, _ = ops.raycast(grid, o, (targets - o).contiguous())
        assert (face >= 0).all(), int((face < 0).sum())
        g = torch.Generator(device="cuda").manual_seed(1)
        d = torch.randn(200_000, 3, generator=g, device="cuda")
        _, face, _ = ops.raycast(grid, p.expand_as(d).contiguous(), d)
        assert (face >= 0).all()


def test_first_and_last_hit_on_a_sphere():
    from sparf_b200 import ops
    n, r = 40, 15.0
    c = (n - 1) / 2 + 0.13
    v, f = TMD._sphere(n, r)
    g = torch.Generator(device="cuda").manual_seed(3)
    o = c + 40.0 * _unit(torch.randn(20000, 3, generator=g, device="cuda"))
    aim = c + 12.0 * (torch.rand(20000, 3, generator=g, device="cuda") * 2 - 1)
    d = aim - o
    grid = ops.distance_grid(v, f)
    t, face, _ = ops.raycast(grid, o, d)
    # analytic: |o + t d - c|^2 = r^2
    od, dd = (o.double() - c), d.double()
    A, B, C = (dd * dd).sum(1), 2 * (od * dd).sum(1), (od * od).sum(1) - r * r
    disc = B * B - 4 * A * C
    hit = disc > 0
    t_in = (-B - disc.clamp(min=0).sqrt()) / (2 * A)
    t_out = (-B + disc.clamp(min=0).sqrt()) / (2 * A)
    closest = (od - ((od * dd).sum(1) / A)[:, None] * dd).norm(dim=1)   # the ray line's distance from the centre
    inner = hit & (closest < r - 1.0)
    assert (face[inner] >= 0).all() and (face[closest > r + 1.0] < 0).all()
    voxel = 1.0 / dd.norm(dim=1)
    assert ((t.double() - t_in).abs()[inner] <= voxel[inner]).all()
    o2 = (o.double() + (t_out[:, None] + 5.0 * voxel[:, None]) * dd).float()
    t2, face2, _ = ops.raycast(grid, o2[inner].contiguous(), (-d[inner]).contiguous())
    last = t_out[inner] + 5.0 * voxel[inner] - t2.double()
    assert (face2 >= 0).all() and ((last - t_out[inner]).abs() <= voxel[inner]).all()


# ------------------------------------------------------------------------------------------------ 4. analytic maps
def _look(cam, target, H, W, f):
    import common
    pose = torch.from_numpy(common.look_at_w2c(cam, target)).cuda()[None]
    K = torch.tensor([[f, 0, W / 2], [0, f, H / 2], [0, 0, 1]], dtype=torch.float32, device="cuda")
    return pose, K


def test_render_plane_head_on():
    from sparf_b200 import mesh
    n = 60
    gxy = np.stack(np.meshgrid(np.arange(n), np.arange(n), indexing="ij"), -1).reshape(-1, 2).astype(np.float32)
    a = (np.arange(n - 1)[:, None] * n + np.arange(n - 1)[None, :]).reshape(-1)
    f = torch.from_numpy(np.stack([np.stack([a, a + n, a + 1], 1), np.stack([a + 1, a + n, a + n + 1], 1)],
                                  1).reshape(-1, 3).astype(np.int64)).cuda()
    z0 = 3.25
    v = torch.from_numpy(np.concatenate([gxy, np.full((len(gxy), 1), z0, np.float32)], 1)).cuda()
    H, W = 96, 128
    cam = (29.5, 29.5, -20.0)
    pose, K = _look(cam, (29.5, 29.5, 10.0), H, W, f=1.2 * W)
    r = mesh.render(dict(vertices=v, faces=f), pose, K, H, W)
    depth = r["depth"][0]
    assert (r["face"] >= 0).all()
    b = 64 * ULP * (60 + 20)
    assert ((depth - (z0 - cam[2])).abs() <= b).all(), (depth - (z0 - cam[2])).abs().max().item()


def test_render_sphere_depth_and_silhouette():
    from sparf_b200 import camera, mesh
    n, r = 64, 25.0
    c = (n - 1) / 2 + 0.13
    v, f = TMD._sphere(n, r)
    normals = _unit(v - c)
    H, W = 240, 320
    pose, K = _look((c + 20.0, c - 35.0, c + 70.0), (c, c, c), H, W, f=1.6 * W)
    out = mesh.render(dict(vertices=v, faces=f, normals=normals), pose, K, H, W)
    o, d = camera.get_center_and_ray(pose, H, W, K[None])
    od, dd = o[0].double() - c, d[0].double()
    A, B, C = (dd * dd).sum(1), 2 * (od * dd).sum(1), (od * od).sum(1) - r * r
    disc = B * B - 4 * A * C
    t_an = (-B - disc.clamp(min=0).sqrt()) / (2 * A)
    closest = (od - ((od * dd).sum(1) / A)[:, None] * dd).norm(dim=1)
    face, depth = out["face"].reshape(-1), out["depth"].reshape(-1).double()
    rim = (closest - r).abs() <= 1.0
    assert torch.equal((face >= 0)[~rim], (closest < r)[~rim])
    hit = (face >= 0) & (closest < r - 1.0)
    voxel = 1.0 / dd.norm(dim=1)
    assert ((depth - t_an).abs()[hit] <= voxel[hit]).all()
    assert torch.isinf(depth[face < 0]).all()
    nm = out["normals"].reshape(-1, 3)
    assert torch.isnan(nm[face < 0]).all() and (_unit(nm[hit]) * _unit((od + t_an[:, None] * dd)[hit].float())).sum(1).min() > 0.98


# ------------------------------------------------------------------------------------------------ 5. culling
def _axis_cams(c, dist, H, W, f):
    import common
    poses = []
    for a in range(3):
        for s in (1, -1):
            cam = np.full(3, c, np.float64)
            cam[a] += s * dist
            up = (0.0, 0.0, 1.0) if a != 2 else (0.0, 1.0, 0.0)
            poses.append(common.look_at_w2c(cam, (c, c, c), up=up))
    K = torch.tensor([[f, 0, W / 2], [0, f, H / 2], [0, 0, 1]], dtype=torch.float32, device="cuda")
    return torch.from_numpy(np.stack(poses)).cuda(), K


def test_cull_one_camera_keeps_only_front_faces():
    from sparf_b200 import mesh
    n, r = 40, 15.0
    c = (n - 1) / 2 + 0.13
    v, f = TMD._sphere(n, r)
    cam = torch.tensor([c + 50.0, c - 10.0, c + 5.0], device="cuda")
    pose, K = _look(tuple(cam.tolist()), (c, c, c), 200, 200, 300.0)
    vis = mesh.visible_faces(dict(vertices=v, faces=f), pose, K, 200, 200)
    nrm = _normals(v, f).double()
    cen = v[f].mean(1).double()
    sign = torch.sign(((cen - c) * nrm).sum(1).sum())        # the extractor's orientation: outward or inward
    facing = sign * (nrm * (cam.double() - cen)).sum(1)
    assert vis.sum() > 100
    assert (facing[vis] >= -1e-6 * (nrm.norm(dim=1) * (cam.double() - cen).norm(dim=1))[vis]).all()


def test_cull_nested_spheres_loses_the_inner_one():
    from sparf_b200 import mesh
    n = 48
    c = (n - 1) / 2 + 0.13
    vo, fo = TMD._sphere(n, 18.0)
    vi, fi = TMD._sphere(n, 8.0)
    v, f = torch.cat([vo, vi]), torch.cat([fo, fi + vo.shape[0]])
    pose, K = _axis_cams(c, 60.0, 256, 256, 400.0)
    st = {}
    out = mesh.cull(dict(vertices=v, faces=f), pose, K, 256, 256, stats=st)
    vis = mesh.visible_faces(dict(vertices=v, faces=f), pose, K, 256, 256)
    assert not vis[fo.shape[0]:].any() and vis[:fo.shape[0]].sum() > 0.9 * fo.shape[0]
    assert out["vertices"].shape[0] <= vo.shape[0] and st["faces_after"] == int(vis.sum())
    assert st == dict(faces_before=f.shape[0], faces_after=int(vis.sum()), views=6, pixels=6 * 256 * 256)


def test_cull_six_views_keep_every_face():
    from sparf_b200 import mesh
    n, r = 10, 3.3
    c = (n - 1) / 2 + 0.13
    v, f = TMD._sphere(n, r)
    pose, K = _axis_cams(c, 12.0, 2048, 2048, 3000.0)
    vis = mesh.visible_faces(dict(vertices=v, faces=f), pose, K, 2048, 2048)
    area = _normals(v, f).norm(dim=1) / 2
    print("%d faces, %d visible, %d below 0.01 voxel^2" % (f.shape[0], vis.sum(), (area < 0.01).sum()))
    assert vis[area >= 0.01].all()


def test_cull_half_mask():
    from sparf_b200 import mesh
    n, r = 40, 15.0
    c = (n - 1) / 2 + 0.13
    v, f = TMD._sphere(n, r)
    H, W = 120, 160
    pose, K = _axis_cams(c, 50.0, H, W, 200.0)
    m = dict(vertices=v, faces=f)
    masks = torch.zeros(6, H, W, dtype=torch.bool, device="cuda")
    masks[:, :, : W // 2] = True
    vis = mesh.visible_faces(m, pose, K, H, W, masks=masks)
    fm = mesh.render(m, pose, K, H, W)["face"]
    want = torch.zeros(f.shape[0], dtype=torch.bool, device="cuda")
    sel = fm[:, :, : W // 2]
    want[sel[sel >= 0]] = True
    assert torch.equal(vis, want)
    assert torch.equal(mesh.visible_faces(m, pose, K, H, W, masks=masks.to(torch.uint8)), want)
    full = mesh.visible_faces(m, pose, K, H, W)
    assert full.sum() > vis.sum()


def test_cull_matches_a_numpy_restatement():
    from sparf_b200 import mesh
    v, f = TMD._torus(40, 11.0, 5.0)
    g = torch.Generator(device="cuda").manual_seed(0)
    m = dict(vertices=v, faces=f, normals=torch.randn(v.shape[0], 3, generator=g, device="cuda"),
             colors=torch.rand(v.shape[0], 3, generator=g, device="cuda"), label="torus")
    c = (40 - 1) / 2 + 0.11
    pose, K = _look((c + 5.0, c - 60.0, c + 25.0), (c, c, c), 150, 200, 250.0)
    vis = mesh.visible_faces(m, pose, K, 150, 200).cpu().numpy()
    out = mesh.cull(m, pose, K, 150, 200)
    fn = f.cpu().numpy()
    kept = fn[vis]
    used = np.zeros(v.shape[0], bool)
    used[kept.reshape(-1)] = True
    new_id = np.cumsum(used) - 1
    assert np.array_equal(out["faces"].cpu().numpy(), new_id[kept])
    for k in ("vertices", "normals", "colors"):
        assert out[k].cpu().numpy().tobytes() == m[k].cpu().numpy()[used].tobytes(), k
    assert out["label"] == "torus" and 0 < vis.sum() < len(fn)


def test_cull_the_extractors_meshes():
    import common
    from sparf_b200 import mesh, tsdf
    from sparf_b200.renderer import Graph
    opt, (_, blobs) = TMC._nerfs(res=64)
    poses, Kc = TMC._ring_cams(6, 60, 80)
    pose, K = torch.from_numpy(poses).cuda(), torch.from_numpy(Kc).cuda()
    meshes = dict(dense=mesh.extract_mesh(opt, blobs, normals=True), sparse=mesh.extract_mesh_sparse(opt, blobs))
    gopt = common.make_opt(fine=True, depth_range=(1.5, 4.5))
    graph = Graph(gopt, torch.device("cuda"))
    for net in graph.get_network_components():
        net.load_state_dict({k: v.cuda() for k, v in TMC.blob_weights(gopt, [TMC.MAIN_TSDF]).items()})
    vol = tsdf.TSDFVolume(res=64)
    tsdf.fuse_renders(gopt, graph, vol, pose, K, 60, 80, (1.5, 4.5))
    meshes["tsdf"] = tsdf.extract_mesh(vol)
    for name, m in meshes.items():
        st = {}
        out = mesh.cull(m, pose, K, 60, 80, stats=st)
        F, V = out["faces"].shape[0], out["vertices"].shape[0]
        assert 0 < F < m["faces"].shape[0], name
        assert out["faces"].min().item() >= 0 and out["faces"].max().item() < V, name
        assert all(out[k].shape[0] == V for k in ("normals", "colors") if k in out)
        res = mesh.compare(out, m, threshold=0.05, n_samples=20_000)
        assert res["accuracy"] < 1e-4 and res["precision"] == 1.0, (name, res)
        print("%s: faces %d -> %d" % (name, st["faces_before"], st["faces_after"]))


# ------------------------------------------------------------------------------------------------ 6. capture, empty
def test_capture_and_replay():
    from sparf_b200 import ops
    v, f = TMD._torus(40, 11.0, 5.0)
    grid = ops.distance_grid(v, f)
    g = torch.Generator(device="cuda").manual_seed(0)
    o = 20.0 + 30.0 * _unit(torch.randn(50_000, 3, generator=g, device="cuda"))
    d = 20.0 + 8.0 * torch.randn(50_000, 3, generator=g, device="cuda") - o
    eager = ops.raycast(grid, o, d, 0.0, 100.0)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.raycast(grid, o, d, 0.0, 100.0)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = ops.raycast(grid, o, d, 0.0, 100.0)
    graph.replay()
    torch.cuda.synchronize()
    assert _same(out, eager)
    o.copy_(20.0 + 25.0 * _unit(torch.randn(50_000, 3, generator=g, device="cuda")))
    graph.replay()
    again = ops.raycast(grid, o, d, 0.0, 100.0)
    torch.cuda.synchronize()
    assert _same(out, again) and (again[1] >= 0).any() and (again[1] < 0).any()


def test_empty_cases():
    from sparf_b200 import mesh, ops
    o, d = torch.rand(10, 3, device="cuda"), torch.rand(10, 3, device="cuda")
    for v in (torch.zeros(0, 3, device="cuda"), torch.rand(5, 3, device="cuda")):
        grid = ops.distance_grid(v, torch.zeros(0, 3, dtype=torch.int64, device="cuda"))
        t, face, bary = ops.raycast(grid, o, d)
        assert torch.isinf(t).all() and (face == -1).all() and torch.isnan(bary).all()
    v, f = TMD._sphere(14, 4.3)
    grid = ops.distance_grid(v, f)
    t, face, bary = ops.raycast(grid, o[:0], d[:0])
    assert t.shape == (0,) and face.shape == (0,) and bary.shape == (0, 3)
    t, face, bary = ops.raycast(grid, o + 100.0, d)                 # every ray misses
    assert torch.isinf(t).all() and (face == -1).all() and torch.isnan(bary).all()
    m = dict(vertices=v[:0], faces=f[:0], colors=v[:0])
    pose, K = _look((0.0, 0.0, -5.0), (0.0, 0.0, 0.0), 4, 6, 5.0)
    r = mesh.render(m, pose, K, 4, 6)
    assert torch.isinf(r["depth"]).all() and (r["face"] == -1).all() and torch.isnan(r["colors"]).all()
    out = mesh.cull(m, pose, K, 4, 6)
    assert out["faces"].shape == (0, 3) and out["vertices"].shape == (0, 3)


# ------------------------------------------------------------------------------------------------ 7. scale
def test_six_million_faces_three_dtu_views():
    from sparf_b200 import camera, ops
    n, r = 880, 420.0
    c = (n - 1) / 2 + 0.13
    v, f = TMD._sphere_on_device(n, r)
    assert f.shape[0] > 6_000_000
    H, W = 1200, 1600
    import common
    poses = [common.look_at_w2c((c + 1100.0 * math.cos(a), c + 1100.0 * math.sin(a), c + 300.0), (c + 40, c - 30, c))
             for a in (0.2, 2.3, 4.4)]
    pose = torch.from_numpy(np.stack(poses)).cuda()
    K = torch.tensor([[1.1 * W, 0, W / 2], [0, 1.1 * W, H / 2], [0, 0, 1]], dtype=torch.float32, device="cuda")
    o, d = camera.get_center_and_ray(pose, H, W, K.expand(3, 3, 3))
    o, d = o.reshape(-1, 3).contiguous(), d.reshape(-1, 3).contiguous()
    grid = ops.distance_grid(v, f)
    got = ops.raycast(grid, o, d)
    half = ops.distance_grid(v, f, cells_per_axis=tuple(max(1, x // 2) for x in grid.dims))
    assert _same(ops.raycast(half, o, d), got)
    t, face, _ = got
    od, dd = o.double() - c, d.double()
    A, B, C = (dd * dd).sum(1), 2 * (od * dd).sum(1), (od * od).sum(1) - r * r
    disc = B * B - 4 * A * C
    t_an = (-B - disc.clamp(min=0).sqrt()) / (2 * A)
    closest = (od - ((od * dd).sum(1) / A)[:, None] * dd).norm(dim=1)
    inner = closest < r - 1.0
    assert inner.any() and (closest > r + 1.0).any()
    assert (face[inner] >= 0).all() and (face[closest > r + 1.0] < 0).all()
    voxel = 1.0 / dd.norm(dim=1)
    assert ((t.double() - t_an).abs()[inner] <= voxel[inner]).all()
    print("6 M faces: grid %s, %d rays, %d hits" % (grid.dims, o.shape[0], int((face >= 0).sum())))


# ------------------------------------------------------------------------------------------------ 8. the tools
def _camera_file(path, pose, K, H, W, mask=None):
    cams = dict(pose_w2c=pose.cpu().numpy(), intr=K.expand(pose.shape[0], 3, 3).cpu().numpy(), H=H, W=W)
    if mask is not None:
        cams["mask"] = mask.cpu().numpy()
    np.savez(path, **cams)


def test_compare_tool_cull(tmp_path, capsys):
    from sparf_b200 import mesh
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import compare_mesh as tool
    n, r = 40, 15.0
    c = (n - 1) / 2 + 0.13
    v, f = TMD._sphere(n, r)
    v2, f2 = TMD._sphere(50, 19.0)
    v2 = (v2 - 24.5) * (15.0 / 19.0) + 19.5
    mesh.write_ply(tmp_path / "p.ply", v, f)
    mesh.write_ply(tmp_path / "r.ply", v2, f2)
    pose, K = _look((c + 50.0, c, c), (c, c, c), 100, 120, 150.0)
    mask = torch.ones(1, 100, 120, dtype=torch.bool)
    mask[:, :50] = False
    _camera_file(tmp_path / "cams.npz", pose, K, 100, 120, mask)
    got = tool.main([str(tmp_path / "p.ply"), str(tmp_path / "r.ply"), "--threshold", "0.1", "--samples", "50000",
                     "--cull", str(tmp_path / "cams.npz")])
    pred = mesh.read_ply(tmp_path / "p.ply")
    pred = {k: x.cuda() for k, x in pred.items()}
    st = {}
    culled = mesh.cull(pred, pose, K[None], 100, 120, masks=mask.cuda(), stats=st)     # the file's intr shape
    ref = mesh.compare(culled, dict(vertices=v2, faces=f2), 0.1, n_samples=50_000)
    assert got == ref
    out = capsys.readouterr().out
    assert "faces %d -> %d (removed %d)" % (st["faces_before"], st["faces_after"],
                                            st["faces_before"] - st["faces_after"]) in out
    assert "cull" in out.splitlines()[-1] and "accuracy %.6g" % ref["accuracy"] in out


def test_extract_mesh_tool_cull(tmp_path):
    from sparf_b200 import mesh
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import extract_mesh as tool
    opt, (_, blobs) = TMC._nerfs(res=64)
    ckpt = str(tmp_path / "model.pth.tar")
    torch.save({"state_dict": {"nerf." + k: v for k, v in blobs.state_dict().items()}}, ckpt)
    poses, Kc = TMC._ring_cams(3, 60, 80)
    pose, K = torch.from_numpy(poses).cuda(), torch.from_numpy(Kc).cuda()
    _camera_file(tmp_path / "cams.npz", pose, K[0], 60, 80)
    out = str(tmp_path / "tool.ply")
    tool.main([ckpt, "--res", "64", "--thres", str(TMC.ISO), "--normals", "--cull", str(tmp_path / "cams.npz"),
               "--out", out])
    m = mesh.cull(mesh.extract_mesh(opt, blobs), pose, K, 60, 80)
    m["normals"] = mesh.density_normals(blobs, m["vertices"])
    ref = str(tmp_path / "ref.ply")
    mesh.write_ply(ref, m["vertices"], m["faces"], m["normals"])
    with open(out, "rb") as a, open(ref, "rb") as b:
        assert a.read() == b.read()
