"""GPU tests of the closest-point queries (csrc/mesh_distance.cu) and mesh.compare: agreement with the fp64 oracle
(tests/mesh_distance_oracle.py) on marching-cubes spheres and tori, an open grid and a degenerate soup; identical bytes
for every grid resolution; analytic geometry; the project's meshes; a 6 M-face mesh; CUDA-graph capture; empty cases
and the tool."""
import math
import os
import sys

import numpy as np
import pytest
import torch

import mesh_distance_oracle as MD
import test_mesh_components as TMC

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ULP = 2.0 ** -24


def _mc(vol):
    from sparf_b200 import ops
    return ops.marching_cubes(torch.from_numpy(np.ascontiguousarray(vol, np.float32)).cuda(), 0.0)


def _sphere(n, r):
    return _mc(TMC._ball((n,) * 3, ((n - 1) / 2 + 0.13,) * 3, r))


def _sphere_on_device(n, r):
    """_sphere for volumes too large to build on the host"""
    from sparf_b200 import ops
    t = torch.arange(n, device="cuda", dtype=torch.float32) - np.float32((n - 1) / 2 + 0.13)
    vol = torch.empty(n, n, n, device="cuda")
    for i in range(n):
        vol[i] = r - torch.sqrt(t[i] ** 2 + t[:, None] ** 2 + t[None, :] ** 2)
    return ops.marching_cubes(vol, 0.0)


def _torus(n, R, r):
    c = (n - 1) / 2 + 0.11
    return _mc(TMC._torus((n,) * 3, (c, c, c), R, r))


def _grid(n, jitter=0.2, seed=0):
    """an open n x n vertex grid with jittered heights, two triangles per cell"""
    rng = np.random.default_rng(seed)
    g = np.stack(np.meshgrid(np.arange(n), np.arange(n), indexing="ij"), -1).reshape(-1, 2).astype(np.float32)
    g += rng.uniform(-jitter, jitter, g.shape).astype(np.float32)
    z = rng.uniform(-0.3, 0.3, (len(g), 1)).astype(np.float32)
    a = (np.arange(n - 1)[:, None] * n + np.arange(n - 1)[None, :]).reshape(-1)
    f = np.stack([np.stack([a, a + n, a + 1], 1), np.stack([a + 1, a + n, a + n + 1], 1)], 1).reshape(-1, 3)
    return torch.from_numpy(np.concatenate([g, z], 1)).cuda(), torch.from_numpy(f.astype(np.int64)).cuda()


def _soup():
    """a jittered grid plus zero-area, collinear and repeated-id faces, duplicates of a face, and unused vertices"""
    v, f = _grid(10, seed=3)
    V = v.shape[0]
    extra_v = torch.tensor([[2.0, 2.0, 3.0], [4.0, 4.0, 3.0], [6.0, 6.0, 3.0], [3.0, 7.0, -2.0], [30.0, 30.0, 30.0]],
                           device="cuda")
    extra_f = torch.tensor([[V, V + 1, V + 2], [V + 2, V, V + 1], [V + 3, V + 3, V + 3], [V + 3, V + 3, 5],
                            [7, 7, 40], [12, 13, 23], [12, 13, 23]], dtype=torch.int64, device="cuda")
    return torch.cat([v, extra_v]), torch.cat([f, extra_f])


MESHES = {"sphere": lambda: _sphere(14, 4.3), "torus": lambda: _torus(18, 5.0, 2.2), "grid": lambda: _grid(16),
          "soup": _soup}


def _surface_points(v, f, n, seed):
    from sparf_b200 import mesh
    return mesh.sample_surface(dict(vertices=v, faces=f), n, seed=seed)


def _queries(v, f, seed=0):
    """{kind: points [n, 3]}: on the surface, near it, far beyond the box, and on the vertices"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    on = _surface_points(v, f, 1500, seed)
    lo, hi = v.min(0).values, v.max(0).values
    ext = (hi - lo).max().item()
    near = on + 0.3 * torch.randn(on.shape, generator=g, device="cuda")
    far = lo + (hi - lo) * (torch.rand(800, 3, generator=g, device="cuda") * 4 - 1.5)
    return dict(on=on, near=near, far=far, vertices=v.clone()), ext


def _bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def _bound(p, v):
    return 16 * ULP * (p.abs().max(1).values.double().cpu().numpy() + v.abs().max().item())


def _check_against_oracle(v, f, p, max_dist=float("inf"), literal=False, grid=None):
    """dist within the bound of the oracle's, index its argmin unless the returned triangle is within the bound of the
    minimum, closest on the returned triangle and at the returned distance (and, with literal, within the bound of the
    oracle's closest point), misses exactly inf / -1 / NaN"""
    from sparf_b200 import ops
    grid = grid or ops.distance_grid(v, f)
    d, i, q = (t.cpu().numpy() for t in ops.closest_points(grid, p, max_dist))
    vn, fn, pn = v.cpu().numpy().astype(np.float64), f.cpu().numpy(), p.cpu().numpy().astype(np.float64)
    d64, i64, q64 = MD.closest_triangles(pn, vn, fn, max_dist)
    b = _bound(p, v)
    hit = i >= 0
    miss64 = i64 < 0
    # a miss is exact; a point within the bound of max_dist may fall on either side
    border = np.abs(d64 - max_dist) <= b if math.isfinite(max_dist) else np.zeros_like(hit)
    assert (hit == ~miss64)[~border].all()
    m = ~hit
    assert np.isinf(d[m]).all() and (d[m] > 0).all() and (i[m] == -1).all() and np.isnan(q[m]).all()
    h = hit & ~miss64
    assert (np.abs(d[h] - d64[h]) <= b[h]).all(), np.max(np.abs(d[h] - d64[h]) / b[h])
    dr, qr = MD.triangle_distance(pn[h], vn, fn, i[h])
    assert ((i[h] == i64[h]) | (dr - d64[h] <= b[h])).all()
    on_tri, _ = MD.triangle_distance(q[h].astype(np.float64), vn, fn, i[h])
    assert (on_tri <= b[h]).all(), np.max(on_tri / b[h])
    assert (np.abs(np.linalg.norm(pn[h] - q[h], axis=1) - dr) <= b[h]).all()
    if literal:
        assert (np.abs(q[h] - qr).max(1) <= b[h]).all(), np.max(np.abs(q[h] - qr).max(1) / b[h])
    return d, i, q


# ------------------------------------------------------------------------------------------------ 1. oracle agreement
@pytest.mark.parametrize("name", sorted(MESHES))
def test_matches_oracle(name):
    v, f = MESHES[name]()
    qs, ext = _queries(v, f)
    for kind, p in qs.items():
        # the closest point of a query far from its triangle is ill-conditioned where two candidates nearly tie: it
        # is checked on its triangle and at its distance, and against the oracle's point where it is well posed
        _check_against_oracle(v, f, p, literal=kind in ("on", "vertices"))
        _check_against_oracle(v, f, p, max_dist=0.1 * ext)


def test_points_match_oracle():
    from sparf_b200 import ops
    v, f = _sphere(40, 15.0)
    qs, ext = _queries(v, f, seed=1)
    pts = _surface_points(v, f, 20000, seed=5)
    grid = ops.distance_grid(pts)
    pn = pts.cpu().numpy().astype(np.float64)
    for kind, p in qs.items():
        for md in (float("inf"), 0.05 * ext):
            d, i, q = ops.closest_points(grid, p, md)
            d, i, q = d.cpu().numpy(), i.cpu().numpy(), q.cpu().numpy()
            d64, i64, _ = MD.closest_vertices(p.cpu().numpy(), pn, md)
            b = _bound(p, pts)
            hit = i >= 0
            border = np.abs(d64 - md) <= b
            assert (hit == (i64 >= 0))[~border].all()
            hit &= i64 >= 0
            assert (np.abs(d[hit] - d64[hit]) <= b[hit]).all()
            dr = np.linalg.norm(p.cpu().numpy()[hit].astype(np.float64) - pn[i[hit]], axis=1)
            assert (dr - d64[hit] <= b[hit]).all()
            assert np.array_equal(q[hit], pts.cpu().numpy()[i[hit]])
            assert np.isinf(d[i < 0]).all() and np.isnan(q[i < 0]).all()


# ------------------------------------------------------------------------------------------------ 2. exactness
@pytest.mark.parametrize("name", sorted(MESHES) + ["points"])
def test_same_bytes_for_every_grid(name):
    from sparf_b200 import ops
    if name == "points":
        v, f = _sphere(30, 11.0)
        v, f = _surface_points(v, f, 1000, 2), None
        qs, _ = _queries(*_sphere(30, 11.0))
    else:
        v, f = MESHES[name]()
        qs, _ = _queries(v, f)
    p = torch.cat(list(qs.values()))
    default = ops.distance_grid(v, f)
    ref = ops.closest_points(default, p)
    cells = [1, 3, 17, None, tuple(4 * d for d in default.dims)]
    for c in cells:
        g = ops.distance_grid(v, f, cells_per_axis=c)
        for _ in range(2):
            got = ops.closest_points(g, p)
            for a, b in zip(got, ref):
                assert torch.equal(_bits(a), _bits(b)), c
    print("%s: default grid %s, %d entries" % (name, default.dims, default.entries))


# ------------------------------------------------------------------------------------------------ 3. analytic geometry
def test_compare_with_itself():
    from sparf_b200 import mesh
    v, f = _sphere(64, 25.0)
    m = dict(vertices=v, faces=f)
    ext = (v.max(0).values - v.min(0).values).max().item()
    r = mesh.compare(m, m, threshold=1e-3 * ext, n_samples=200_000)
    assert r["accuracy"] < 1e-6 * ext and r["completeness"] < 1e-6 * ext and r["fscore"] == 1.0
    assert r["n_pred"] == r["n_ref"] == 200_000


def test_shifted_plane():
    from sparf_b200 import mesh, ops
    n, delta = 60, 0.37
    g = np.stack(np.meshgrid(np.arange(n), np.arange(n), indexing="ij"), -1).reshape(-1, 2).astype(np.float32)
    a = (np.arange(n - 1)[:, None] * n + np.arange(n - 1)[None, :]).reshape(-1)
    f = torch.from_numpy(np.stack([np.stack([a, a + n, a + 1], 1), np.stack([a + 1, a + n, a + n + 1], 1)],
                                  1).reshape(-1, 3).astype(np.int64)).cuda()
    v0 = torch.from_numpy(np.concatenate([g, np.zeros((len(g), 1), np.float32)], 1)).cuda()
    v1 = v0.clone()
    v1[:, 2] = delta
    pred, ref = dict(vertices=v1, faces=f), dict(vertices=v0, faces=f)
    pts = mesh.sample_surface(pred, 100_000, seed=1)
    d, _, q = ops.closest_points(ops.distance_grid(v0, f), pts)
    b = _bound(pts, v1)
    assert (np.abs(d.cpu().numpy() - delta) <= b).all()
    assert (q[:, 2] == 0).all()
    assert mesh.compare(pred, ref, 1.01 * delta, n_samples=100_000)["fscore"] == 1.0
    assert mesh.compare(pred, ref, 0.99 * delta, n_samples=100_000)["fscore"] == 0.0


def test_sphere_against_analytic_points():
    """a marching-cubes sphere against 1 M points on the analytic sphere: every distance is at least the samples'
    analytic |(|v - c| - r)| (no point of the sphere is nearer), and the mean exceeds its mean by at most the points'
    spacing"""
    from sparf_b200 import mesh
    n, r = 96, 40.0
    c = (n - 1) / 2 + 0.13
    v, f = _sphere(n, r)
    g = torch.Generator(device="cuda").manual_seed(7)
    u = torch.randn(1_000_000, 3, generator=g, device="cuda", dtype=torch.float64)
    cloud = (c + r * u / u.norm(dim=1, keepdim=True)).float()
    pred = mesh.prepare(dict(vertices=v, faces=f), n_samples=1_000_000, seed=0)
    res = mesh.compare(pred, dict(vertices=cloud), threshold=0.5)
    analytic = ((pred["points"].double() - c).norm(dim=1) - r).abs()
    bound = 16 * ULP * 2 * n
    spacing = math.sqrt(4 * math.pi * r * r / 1e6)
    assert res["accuracy"] >= analytic.mean().item() - bound
    assert res["accuracy"] <= analytic.mean().item() + spacing
    print("accuracy %.5f, analytic %.5f, spacing %.4f" % (res["accuracy"], analytic.mean().item(), spacing))


# ------------------------------------------------------------------------------------------------ 4. project meshes
def test_simplified_sphere_hausdorff():
    from sparf_b200 import mesh
    n, r = 384, 175.0
    v, f = _sphere(n, r)
    assert f.shape[0] > 1_100_000
    m = dict(vertices=v, faces=f)
    s = mesh.simplify(m, f.shape[0] // 100)
    res = mesh.compare(s, m, threshold=0.25, n_samples=1_000_000)
    print("simplified to %d faces: hausdorff %.4f, chamfer %.5f voxels" % (s["faces"].shape[0], res["hausdorff"],
                                                                          res["chamfer"]))
    assert res["hausdorff"] < 0.5


def _blob_nerf(opt):
    from sparf_b200.frequency_nerf import NeRF
    nerf = NeRF(opt).cuda()
    nerf.load_state_dict({k: v.cuda() for k, v in TMC.blob_weights(opt, [TMC.MAIN_TSDF]).items()})
    return nerf


def test_dense_against_sparse_extraction():
    import common
    from sparf_b200 import mesh
    from sparf_b200.utils.edict import edict
    opt = common.make_opt()
    opt.trimesh = edict(res=128, range=[-1.2, 1.2], thres=TMC.ISO)
    nerf = _blob_nerf(opt)
    dense, sparse = mesh.extract_mesh(opt, nerf), mesh.extract_mesh_sparse(opt, nerf)
    assert torch.equal(dense["faces"], sparse["faces"]) and torch.equal(dense["vertices"], sparse["vertices"])
    res = mesh.compare(dense, sparse, threshold=1e-3, n_samples=200_000)
    assert res["chamfer"] < 1e-6 * 2.4 and res["fscore"] == 1.0


def test_tsdf_against_dense():
    import common
    from sparf_b200 import mesh, tsdf
    from sparf_b200.renderer import Graph
    from sparf_b200.utils.edict import edict
    opt = common.make_opt(fine=True, depth_range=(1.5, 4.5))
    graph = Graph(opt, torch.device("cuda"))
    for net in graph.get_network_components():
        net.load_state_dict({k: v.cuda() for k, v in TMC.blob_weights(opt, [TMC.MAIN_TSDF]).items()})
    poses, Kc = TMC._ring_cams(12, 60, 80)
    vol = tsdf.TSDFVolume(res=64)
    tsdf.fuse_renders(opt, graph, vol, torch.from_numpy(poses), torch.from_numpy(Kc), 60, 80, (1.5, 4.5))
    fused = tsdf.extract_mesh(vol)
    opt.trimesh = edict(res=128, range=[-1.2, 1.2], thres=TMC.ISO)
    dense = mesh.extract_mesh(opt, graph.nerf_fine)
    assert fused["faces"].shape[0] and dense["faces"].shape[0]
    res = mesh.compare(fused, dense, threshold=0.05, n_samples=200_000)
    print("TSDF against dense: %s" % res)
    assert all(math.isfinite(res[k]) for k in ("accuracy", "completeness", "chamfer", "hausdorff", "fscore"))


# ------------------------------------------------------------------------------------------------ 5. scale
def test_six_million_faces():
    from sparf_b200 import mesh, ops
    n, r = 880, 420.0
    v, f = _sphere_on_device(n, r)
    assert f.shape[0] > 6_000_000
    pts = _surface_points(*_sphere_on_device(n - 80, r - 38.0), 1_000_000, seed=3) + 40.0
    grid = ops.distance_grid(v, f)
    d, i, q = ops.closest_points(grid, pts)
    torch.cuda.synchronize()
    assert (i >= 0).all()
    g = torch.Generator(device="cpu").manual_seed(0)
    sel = torch.randperm(pts.shape[0], generator=g)[:2000].cuda()
    p = pts[sel]
    b = _bound(p, v)
    dn = d[sel].cpu().numpy().astype(np.float64)
    d64, i64, _ = MD.closest_triangles_near(p.cpu().numpy().astype(np.float64), v.cpu().numpy().astype(np.float64),
                                            f.cpu().numpy(), dn + b)
    assert (i64 >= 0).all()
    assert (np.abs(dn - d64) <= b).all()
    print("6 M faces: grid %s, %d entries; mean distance %.4f" % (grid.dims, grid.entries, d.mean().item()))


# ------------------------------------------------------------------------------------------------ 6. capture
def test_capture_and_replay():
    from sparf_b200 import ops
    v, f = _torus(40, 11.0, 5.0)
    grid = ops.distance_grid(v, f)
    p = _surface_points(v, f, 50_000, 1) + 0.2
    eager = ops.closest_points(grid, p, 3.0)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.closest_points(grid, p, 3.0)          # warm-up off the default stream
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = ops.closest_points(grid, p, 3.0)
    graph.replay()
    torch.cuda.synchronize()
    for a, b in zip(out, eager):
        assert torch.equal(a.nan_to_num(), b.nan_to_num())
    p.copy_(_surface_points(v, f, 50_000, 2) * 1.1)
    graph.replay()
    again = ops.closest_points(grid, p, 3.0)
    torch.cuda.synchronize()
    for a, b in zip(out, again):
        assert torch.equal(a.nan_to_num(), b.nan_to_num())
    assert (again[1] == -1).any() and (again[1] >= 0).any()


# ------------------------------------------------------------------------------------------------ 7. empty cases, tool
def test_empty_cases():
    from sparf_b200 import mesh, ops
    p = torch.rand(10, 3, device="cuda")
    for v, f in ((torch.zeros(0, 3, device="cuda"), None), (torch.zeros(0, 3, device="cuda"),
                                                          torch.zeros(0, 3, dtype=torch.int64, device="cuda")),
                 (torch.rand(5, 3, device="cuda"), torch.zeros(0, 3, dtype=torch.int64, device="cuda"))):
        g = ops.distance_grid(v, f)
        assert g.entries == 0 and g.cell_start.tolist() == [0]
        d, i, q = ops.closest_points(g, p)
        assert torch.isinf(d).all() and (i == -1).all() and torch.isnan(q).all()
        d, i, q = ops.closest_points(g, p[:0])
        assert d.shape == (0,) and i.shape == (0,) and q.shape == (0, 3)
    v, f = _sphere(14, 4.3)
    g = ops.distance_grid(v, f)
    d, i, q = ops.closest_points(g, p[:0])
    assert d.shape == (0,) and q.shape == (0, 3)
    m = dict(vertices=v, faces=f)
    empty = dict(vertices=v[:0], faces=f[:0])
    r = mesh.compare(empty, m, threshold=1.0, n_samples=1000)
    assert math.isnan(r["accuracy"]) and r["completeness"] == float("inf") and r["fscore"] == 0.0
    assert r["precision"] == 0.0 and r["recall"] == 0.0 and r["n_pred"] == 0 and r["n_ref"] == 1000
    r = mesh.compare(m, empty, threshold=1.0, n_samples=1000, max_dist=5.0)
    assert r["accuracy"] == 5.0 and math.isnan(r["completeness"]) and r["hausdorff"] == 5.0 and r["fscore"] == 0.0


def test_compare_tool(tmp_path, capsys):
    from sparf_b200 import mesh
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import compare_mesh as tool
    v, f = _sphere(40, 15.0)
    v2, f2 = _sphere(50, 19.0)
    v2 = (v2 - 24.5) * (15.0 / 19.0) + 19.5
    mesh.write_ply(tmp_path / "p.ply", v, f)
    mesh.write_ply(tmp_path / "r.ply", v2, f2)
    got = tool.main([str(tmp_path / "p.ply"), str(tmp_path / "r.ply"), "--threshold", "0.1", "--samples", "50000"])
    ref = mesh.compare(dict(vertices=v, faces=f), dict(vertices=v2, faces=f2), 0.1, n_samples=50_000)
    assert got == ref
    out = capsys.readouterr().out
    assert "accuracy %.6g" % ref["accuracy"] in out and "fscore %.6g" % ref["fscore"] in out
    assert "V %d, F %d" % (v.shape[0], f.shape[0]) in out and "query" in out
