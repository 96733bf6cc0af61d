"""Marching cubes on the device (sparf_mcubes_count / sparf_mcubes_emit, ops.marching_cubes) against the NumPy oracle
(tests/mcubes_oracle.py), on analytic surfaces and edge cases, under CUDA-graph capture; and the mesh module
(sparf_b200.mesh): density_grid against NeRF.forward, normals, a 513^3 lattice, and tools/extract_mesh.py on a snapshot."""
import ctypes
import os

import numpy as np
import pytest
import torch

import mcubes_oracle as O

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _mc(vol, iso):
    from sparf_b200 import ops
    v, f = ops.marching_cubes(torch.as_tensor(vol).cuda(), iso)
    torch.cuda.synchronize()
    return v.cpu().numpy(), f.cpu().numpy()


def _check_equal(vol, iso):
    vol = np.ascontiguousarray(vol, np.float32)
    v, f = _mc(vol, iso)
    rv, rf = O.marching_cubes(vol, iso)
    assert v.shape == rv.shape and f.shape == rf.shape, (v.shape, rv.shape, f.shape, rf.shape)
    assert np.array_equal(v.view(np.uint32), rv.view(np.uint32)), "vertices differ in %d places" % (v != rv).sum()
    assert np.array_equal(f, rf)
    return v, f


def _gaussians(shape, seed, n=6):
    rng = np.random.default_rng(seed)
    x = np.stack(np.meshgrid(*[np.arange(s, dtype=np.float64) for s in shape], indexing="ij"), -1)
    out = np.zeros(shape)
    for _ in range(n):
        c = rng.random(3) * np.array(shape)
        w = 2 + 6 * rng.random()
        out += rng.uniform(0.5, 1.5) * np.exp(-((x - c) ** 2).sum(-1) / (2 * w * w))
    return out.astype(np.float32)


@pytest.mark.parametrize("shape,seed,iso", [((37, 50, 23), 0, 0.5), ((37, 50, 23), 1, 0.25), ((64, 17, 40), 2, 0.6)])
def test_smooth_volumes_match_oracle(shape, seed, iso):
    v, f = _check_equal(_gaussians(shape, seed), iso)
    assert len(f) > 100


def test_random_and_tied_volumes_match_oracle():
    rng = np.random.default_rng(7)
    for shape in ((20, 17, 31), (2, 9, 3), (33, 2, 2)):
        _check_equal(np.where(rng.random(shape) < 0.5, 1.0, -1.0), 0.0)
    for shape, iso in (((19, 23, 21), 0.0), ((19, 23, 21), 1.0), ((8, 40, 9), -1.0)):
        vol = rng.integers(-2, 3, shape).astype(np.float32)      # exact ties at iso: s = 0 on those edges
        _, f = _check_equal(vol, iso)
        assert len(f)
    vol = rng.standard_normal((15, 16, 17)).astype(np.float32)   # inside points on the border: an open mesh
    _check_equal(vol, 0.3)


def test_single_cell_volumes_match_oracle():
    for c in range(256):
        vol = np.array([1.0 if c >> q & 1 else -1.0 for q in range(8)], np.float32).reshape(2, 2, 2).transpose(2, 1, 0)
        _check_equal(vol * np.float32(0.75) + np.float32(0.1), 0.1)


def test_nerf_lattice_matches_oracle():
    import common
    from sparf_b200 import mesh
    from sparf_b200.frequency_nerf import NeRF
    opt = common.make_opt(barf_c2f=(0.1, 0.5))
    nerf = NeRF(opt).cuda()
    nerf.load_state_dict({k: v.cuda() for k, v in common.det_weights(opt, 3, progress=0.3).items()})
    sigma = mesh.density_grid(opt, nerf, res=64)
    assert sigma.shape == (65, 65, 65)
    iso = sigma.median().item()
    _, f = _check_equal(sigma.cpu().numpy(), iso)
    assert len(f) > 1000


def _field(kind, n=130):
    x = np.stack(np.meshgrid(*[np.arange(n, dtype=np.float64)] * 3, indexing="ij"), -1)
    c = np.array([64.3, 63.7, 64.9])
    if kind == "sphere":
        f = 40.0 - np.linalg.norm(x - c, axis=-1)
    elif kind == "torus":
        d = np.linalg.norm(x[..., :2] - c[:2], axis=-1)
        f = 12.0 - np.sqrt((d - 35.0) ** 2 + (x[..., 2] - c[2]) ** 2)
    else:
        f = np.maximum(20.0 - np.linalg.norm(x - [35.2, 64.1, 63.8], axis=-1), 20.0 - np.linalg.norm(x - [94.6, 64.3, 64.7], axis=-1))
    return f.astype(np.float32), c


@pytest.mark.parametrize("kind,euler", [("sphere", 2), ("torus", 0), ("two_spheres", 4)])
def test_analytic_surfaces(kind, euler):
    """iso-surfaces of signed-distance-like fields on 130^3: closed, oriented, the right Euler characteristic; the
    sphere's area within 1 % of 4 pi r^2 and every face normal pointing away from its centre"""
    vol, c = _field(kind)
    v, f = _mc(vol, 0.0)
    assert len(f) > 1000
    assert O.is_closed_and_oriented(f)
    assert O.euler_characteristic(f) == euler
    if kind == "sphere":
        fn = O.face_normals(v, f)
        area = 0.5 * np.linalg.norm(fn, axis=1).sum()
        assert abs(area / (4 * np.pi * 40.0 ** 2) - 1) < 0.01, area
        assert (np.einsum("ij,ij->i", fn, v[f].mean(1) - c) > 0).all()


def test_edge_cases():
    from sparf_b200 import ops
    for fill in (-1.0, 1.0):
        v, f = ops.marching_cubes(torch.full((9, 10, 11), fill, device="cuda"), 0.0)
        assert v.shape == (0, 3) and f.shape == (0, 3)
    rng = np.random.default_rng(11)
    vol = rng.standard_normal((30, 31, 32)).astype(np.float32)
    bad = rng.random(vol.shape)
    vol[bad < 0.03] = np.nan
    vol[(bad >= 0.03) & (bad < 0.05)] = np.inf
    vol[(bad >= 0.05) & (bad < 0.07)] = -np.inf
    v, f = ops.marching_cubes(torch.from_numpy(vol).cuda(), 0.0)
    v2, f2 = ops.marching_cubes(torch.from_numpy(vol).cuda(), 0.0)
    torch.cuda.synchronize()
    rv, rf = O.marching_cubes(vol, 0.0)
    assert v.shape == rv.shape and f.shape == rf.shape
    assert f.min().item() >= 0 and f.max().item() < v.shape[0]
    assert torch.equal(f, f2) and np.array_equal(v.cpu().numpy().view(np.uint32), v2.cpu().numpy().view(np.uint32))
    with pytest.raises(RuntimeError):
        ops.marching_cubes(torch.zeros(1, 5, 5, device="cuda"), 0.0)


def test_count_emit_capture_and_replay():
    """count + emit captured in one CUDA graph: replays give the eager call's bytes, also on new volume contents"""
    from sparf_b200 import _lib, ops
    L = _lib.lib()
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    shape = (41, 38, 45)
    vols = [torch.from_numpy(_gaussians(shape, s)).cuda() for s in (20, 21)]
    vol = vols[0].clone()
    iso = 0.5
    ref = [ops.marching_cubes(x, iso) for x in vols]
    cap = max(r[0].shape[0] for r in ref), max(r[1].shape[0] for r in ref)
    ws = torch.empty(L.sparf_mcubes_workspace_bytes(*shape), dtype=torch.uint8, device="cuda")
    totals = torch.zeros(2, dtype=torch.int64, device="cuda")
    verts = torch.zeros(cap[0], 3, device="cuda")
    faces = torch.zeros(cap[1], 3, dtype=torch.int64, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=s):
        st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        _lib.check(L.sparf_mcubes_count(p(vol), *shape, iso, p(totals), p(ws), ws.numel(), st), "mcubes_count")
        _lib.check(L.sparf_mcubes_emit(p(vol), *shape, iso, p(verts), p(faces), p(ws), ws.numel(), st), "mcubes_emit")
    for x, (rv, rf) in zip(vols + vols[:1], ref + ref[:1]):
        vol.copy_(x)
        graph.replay()
        torch.cuda.synchronize()
        V, F = totals.tolist()
        assert (V, F) == (rv.shape[0], rf.shape[0])
        assert torch.equal(verts[:V].view(torch.int32), rv.view(torch.int32)) and torch.equal(faces[:F], rf)


@pytest.mark.parametrize("engine", ["simt_fp32", "tc_3x"])
def test_density_grid_matches_nerf_forward(engine):
    """density_grid is NeRF.forward's density_samples at the same lattice points (the bound of
    test_density.test_softplus_of_raw_matches_nerf_forward)"""
    import common
    from sparf_b200 import _lib, mesh, ops
    from sparf_b200.frequency_nerf import NeRF
    if not _lib.lib().sparf_engine_available(_lib.ENGINES[engine]):
        pytest.skip("%s not available" % engine)
    opt = common.make_opt(barf_c2f=(0.1, 0.5))
    nerf = NeRF(opt).cuda()
    nerf.load_state_dict({k: v.cuda() for k, v in common.det_weights(opt, 9, progress=0.3).items()})
    res = 40
    old = mesh.SLAB_POINTS
    mesh.SLAB_POINTS = 5 * 41 * 41 + 7      # several slabs, the last one partial
    try:
        sigma = mesh.density_grid(opt, nerf, res=res, range=(-1.3, 1.1), engine=engine)
    finally:
        mesh.SLAB_POINTS = old
    t = torch.linspace(-1.3, 1.1, res + 1)
    pts = torch.stack(torch.meshgrid(t, t, t, indexing="ij"), dim=-1).cuda().view(1, -1, 1, 3)
    ray = torch.tensor([0.3, -0.5, 0.8], device="cuda").expand(1, pts.shape[1], 3).contiguous()
    prev = ops.get_engine()
    ops.set_engine(engine)
    try:
        with torch.no_grad():
            dens = nerf.forward(opt, pts, ray, None, None)["density_samples"].view(res + 1, res + 1, res + 1)
    finally:
        ops.set_engine(prev)
    assert ((sigma - dens).abs() / dens.abs().clamp_min(1e-30)).max().item() <= 1e-6


def test_extract_mesh_normals_on_a_smooth_field():
    """normals have unit length and agree with the face orientation (toward falling density) on >= 99 % of faces"""
    import common
    from sparf_b200 import mesh
    from sparf_b200.frequency_nerf import NeRF
    from sparf_b200.utils.edict import edict
    opt = common.make_opt(L_3D=2)
    nerf = NeRF(opt).cuda()
    nerf.load_state_dict({k: v.cuda() for k, v in common.det_weights(opt, 4).items()})
    sigma = mesh.density_grid(opt, nerf, res=64)
    opt.trimesh = edict(res=64, range=[-1.2, 1.2], thres=sigma.median().item())
    m = mesh.extract_mesh(opt, nerf, normals=True)
    v, f, n = m["vertices"], m["faces"], m["normals"]
    assert len(f) > 1000 and n.shape == v.shape
    assert ((n.norm(dim=-1) - 1).abs() < 1e-5).all()
    fn = torch.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]], dim=-1)
    agree = ((fn * n[f].mean(1)).sum(-1) > 0).float().mean().item()
    print("normals agree with the face orientation on %.4f of %d faces" % (agree, len(f)))
    assert agree >= 0.99


def test_large_lattice_513():
    """the 513^3 lattice (135 M points) of a NeRF on tc_3x: ids in range, every vertex referenced"""
    import common
    from sparf_b200 import _lib, mesh
    from sparf_b200.frequency_nerf import NeRF
    if not _lib.lib().sparf_engine_available(_lib.ENGINE_TC_3X):
        pytest.skip("tc_3x not available")
    opt = common.make_opt()
    nerf = NeRF(opt).cuda()
    nerf.load_state_dict({k: v.cuda() for k, v in common.det_weights(opt, 5, peaky=True, sigma_bias=-2.0).items()})
    sigma = mesh.density_grid(opt, nerf, res=512, engine="tc_3x")
    assert sigma.shape == (513, 513, 513) and torch.isfinite(sigma).all()
    iso = torch.quantile(sigma.view(-1)[:: 97].float(), 0.9).item()
    v, f = mesh.marching_cubes(sigma, iso)
    torch.cuda.synchronize()
    print("513^3: iso %.4f, V %d, F %d" % (iso, v.shape[0], f.shape[0]))
    assert f.shape[0] > 0 and f.min().item() >= 0 and f.max().item() < v.shape[0]
    used = torch.zeros(v.shape[0], dtype=torch.bool, device="cuda")
    used[f.view(-1)] = True
    assert used.all()
    assert ((v >= 0) & (v <= 512)).all()


def test_extract_mesh_tool_on_a_snapshot(tmp_path):
    """tools/extract_mesh.py on a reference-layout snapshot ({"state_dict": Graph.state_dict()}) of the synthetic
    teacher writes a PLY whose mesh is the library's"""
    import sys
    import common
    from sparf_b200 import mesh
    from sparf_b200.renderer import Graph
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import extract_mesh as tool
    opt = common.make_opt(fine=True)
    graph = Graph(opt, torch.device("cuda"))
    graph.nerf.load_state_dict(common.det_weights(opt, 5, peaky=True, sigma_bias=-2.0, progress=1.0))
    graph.nerf_fine.load_state_dict(common.det_weights(opt, 82, peaky=True, sigma_bias=-2.0, progress=1.0))
    ckpt = str(tmp_path / "model.pth.tar")
    torch.save({"state_dict": graph.state_dict()}, ckpt)
    sigma = mesh.density_grid(opt, graph.nerf_fine, res=48)
    thres = torch.quantile(sigma.view(-1), 0.8).item()
    out = str(tmp_path / "mesh.ply")
    tool.main([ckpt, "--network", "nerf_fine", "--res", "48", "--thres", str(thres), "--normals", "--out", out])
    props, faces = O.read_ply(out)
    opt.trimesh = dict(res=48, range=[-1.2, 1.2], thres=thres)
    ref = mesh.extract_mesh(opt, graph.nerf_fine)
    assert len(faces) > 0 and np.array_equal(faces, ref["faces"].cpu().numpy())
    xyz = np.stack([props[k] for k in "xyz"], 1)
    assert np.array_equal(xyz, ref["vertices"].cpu().numpy())
    nrm = np.stack([props[k] for k in ("nx", "ny", "nz")], 1)
    assert np.abs(np.linalg.norm(nrm, axis=1) - 1).max() < 1e-5
