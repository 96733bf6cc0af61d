"""TSDF fusion on the GPU (sparf_tsdf_integrate, the masked marching cubes, sparf_b200/tsdf.py, tools/extract_mesh.py
--tsdf): the integration against the NumPy oracle (tests/tsdf_oracle.py), the projection convention against the ray
generation, analytic surfaces, the masked marching cubes against the dense one, renders of a Graph, CUDA-graph capture."""
import ctypes
import math
import os
import sys

import numpy as np
import pytest
import torch

import tsdf_oracle as T

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cams(B, H, W, seed, radius=3.0, focal=None, jitter=0.3):
    """B w2c poses on a sphere of `radius` looking at a point near the origin, and one K"""
    import common
    rng = np.random.default_rng(seed)
    poses = []
    for b in range(B):
        d = rng.standard_normal(3)
        d /= np.linalg.norm(d)
        up = (0.0, -1.0, 0.0) if abs(d[1]) < 0.9 else (1.0, 0.0, 0.0)
        poses.append(common.look_at_w2c(radius * d, target=tuple(jitter * rng.uniform(-1, 1, 3)), up=up))
    f = float(focal if focal is not None else 1.2 * max(H, W))
    K = np.array([[f, 0, W / 2.0], [0, f, H / 2.0], [0, 0, 1]], np.float32)
    return np.stack(poses), np.stack([K] * B)


def _random_maps(B, H, W, seed):
    rng = np.random.default_rng(seed)
    depth = rng.uniform(2.0, 4.0, (B, H, W)).astype(np.float32)
    bad = rng.random((B, H, W))
    depth[bad < 0.03] = np.nan
    depth[(bad >= 0.03) & (bad < 0.05)] = np.inf
    depth[(bad >= 0.05) & (bad < 0.07)] = -1.0
    rgb = rng.random((B, H, W, 3)).astype(np.float32)
    valid = rng.random((B, H, W)) < 0.85
    return depth, rgb, valid


def _cuda(*xs):
    return [None if x is None else torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in xs]


# ------------------------------------------------------------------------------------------------ 1. the oracle
@pytest.mark.parametrize("with_rgb,with_valid", [(True, True), (False, False), (True, False)])
def test_integration_matches_oracle(with_rgb, with_valid):
    """random cameras around the box and random maps, integrated in batches of 2, 3 and 4 views: the weights equal the
    oracle's, tsdf and color within 1e-5 of its fp64 averages"""
    from sparf_b200 import tsdf
    B, H, W = 9, 24, 32
    poses, K = _cams(B, H, W, seed=1)
    depth, rgb, valid = _random_maps(B, H, W, seed=2)
    rgb = rgb if with_rgb else None
    valid = valid if with_valid else None
    vol = tsdf.TSDFVolume(res=32, trunc=0.3)
    for b0, b1 in ((0, 2), (2, 5), (5, 9)):
        sl = lambda x: None if x is None else x[b0:b1]
        d, p, k, c, v = _cuda(depth[b0:b1], poses[b0:b1], K[b0:b1], sl(rgb), sl(valid))
        tsdf.integrate_(vol, d, p, k, rgb=c, valid=v)
    torch.cuda.synchronize()
    rt, rw, rc = T.integrate(vol.axis.cpu().numpy(), vol.trunc, poses, K, depth, rgb, valid)
    w = vol.weight.cpu().numpy().reshape(-1)
    assert np.array_equal(w, rw), "weights differ at %d points" % (w != rw).sum()
    assert rw.max() >= 3 and (rw == 0).sum() > 0
    assert np.abs(vol.tsdf.cpu().numpy().reshape(-1) - rt).max() <= 1e-5
    if with_rgb:
        assert np.abs(vol.color.cpu().numpy().reshape(-1, 3) - rc).max() <= 1e-5
    else:
        assert (vol.color == 0).all()


def test_shared_intrinsics_and_batches_agree():
    """intr [3, 3] is every view's K; one call over all views equals any split into consecutive batches, bit for bit"""
    from sparf_b200 import tsdf
    B, H, W = 6, 20, 28
    poses, K = _cams(B, H, W, seed=4)
    depth, rgb, valid = _random_maps(B, H, W, seed=5)
    d, p, k, c, v = _cuda(depth, poses, K, rgb, valid)
    one = tsdf.TSDFVolume(res=40)
    tsdf.integrate_(one, d, p, k[0], rgb=c, valid=v)
    split = tsdf.TSDFVolume(res=40)
    for b in range(B):
        tsdf.integrate_(split, d[b:b + 1], p[b:b + 1], k[b:b + 1], rgb=c[b:b + 1], valid=v[b:b + 1])
    for a in ("tsdf", "weight", "color"):
        assert torch.equal(getattr(one, a), getattr(split, a)), a


# ------------------------------------------------------------------------------------------------ 2. the projection
def test_projection_inverts_raygen():
    """A camera at a lattice point looking along +z with f = D (in voxels) and c = W/2 + 1/2: the ray of pixel (i, j)
    passes through the lattice points c + k (m, l, D) voxels (m = i - W/2, l = j - H/2).  Depth = the ray's own t (from
    ops.raygen) at k = k_ij, random per pixel: those lattice points get s = 0, up to fp32 rounding, and weight 1.  A
    point landing in a neighbouring pixel would read a different k."""
    from sparf_b200 import ops, tsdf
    res, D, H, W = 48, 16, 16, 16
    vol = tsdf.TSDFVolume(res=res, range=(-1.2, 1.2), trunc=0.2)
    h = 2.4 / res
    cidx = np.array([24, 24, 0])
    axis = vol.axis.cpu().numpy().astype(np.float64)
    c = axis[cidx]
    pose = np.array([[[1, 0, 0, -c[0]], [0, 1, 0, -c[1]], [0, 0, 1, -c[2]]]], np.float32)
    K = np.array([[[D, 0, W / 2 + 0.5], [0, D, H / 2 + 0.5], [0, 0, 1]]], np.float32)
    kk = np.random.default_rng(0).integers(1, 3, (H, W))
    jj, ii = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    m, l = ii - W // 2, jj - H // 2
    lat = cidx[None, None] + kk[..., None] * np.stack([m, l, np.full_like(m, D)], -1)     # lattice index [H, W, 3]
    X = axis[lat]                                                                         # world points on the rays
    p, k = _cuda(pose, K)
    o, d = ops.raygen(p, k, W, ray_idx=torch.arange(H * W, device="cuda"))
    o, d = o[0].double().cpu().numpy(), d[0].double().cpu().numpy()
    t = ((X.reshape(-1, 3) - o) * d).sum(-1) / (d * d).sum(-1)
    assert np.abs(o + d * t[:, None] - X.reshape(-1, 3)).max() < 1e-5                   # the rays do pass through X
    depth = torch.from_numpy(t.astype(np.float32).reshape(1, H, W)).cuda()
    tsdf.integrate_(vol, depth, p, k)
    n = res + 1
    lin = (lat[..., 0] * n + lat[..., 1]) * n + lat[..., 2]
    got_t = vol.tsdf.view(-1)[torch.from_numpy(lin.reshape(-1)).cuda()].cpu().numpy()
    got_w = vol.weight.view(-1)[torch.from_numpy(lin.reshape(-1)).cuda()].cpu().numpy()
    assert (got_w == 1).all()
    assert np.abs(got_t * vol.trunc).max() <= 2e-6, np.abs(got_t * vol.trunc).max()
    # one voxel further along z: s = -h; one voxel nearer: s = +h (away from the border, where the nearer point's
    # projection moves by up to |m| / (k D - 1) < 1/2 pixel and stays in pixel (i, j))
    inner = (np.abs(m) <= 6) & (np.abs(l) <= 6)
    for dz, s in ((1, -h), (-1, h)):
        lin2 = lin[inner] + dz
        got = vol.tsdf.view(-1)[torch.from_numpy(lin2.reshape(-1)).cuda()].cpu().numpy()
        assert np.abs(got * vol.trunc - s).max() <= 1e-5


# ------------------------------------------------------------------------------------------------ 3. analytic surfaces
def _ring_cams(n, H, W, radius=3.0, seed=0):
    """n views around the box, at varied heights"""
    import common
    rng = np.random.default_rng(seed)
    poses = []
    for b in range(n):
        a = 2 * math.pi * b / n
        y = rng.uniform(-1.5, 1.5)
        poses.append(common.look_at_w2c((radius * math.sin(a), y, -radius * math.cos(a))))
    f = 1.1 * max(H, W)
    K = np.array([[f, 0, W / 2.0], [0, f, H / 2.0], [0, 0, 1]], np.float32)
    return np.stack(poses), np.stack([K] * n)


def _depth_of(kind, o, d, far=100.0):
    """exact z-depth maps (the ray parameter t of raygen's rays, whose camera-space z is 1) of an analytic surface"""
    o, d = o.double(), d.double()
    if kind[0] == "sphere":
        _, c, r = kind
        c = torch.tensor(c, dtype=torch.float64, device=o.device)
        oc = o - c
        a, b, cc = (d * d).sum(-1), 2 * (oc * d).sum(-1), (oc * oc).sum(-1) - r * r
        disc = b * b - 4 * a * cc
        t = (-b - disc.clamp_min(0).sqrt()) / (2 * a)
        t = torch.where((disc > 0) & (t > 0), t, torch.full_like(t, far))
    else:
        _, nrm, off = kind
        nrm = torch.tensor(nrm, dtype=torch.float64, device=o.device)
        t = (off - (o * nrm).sum(-1)) / (d * nrm).sum(-1)
        t = torch.where(t > 0, t, torch.full_like(t, far))
    return t.float()


def _fuse_analytic(kind, n_views=20, H=64, W=80, res=64, rgb_fn=None):
    from sparf_b200 import ops, tsdf
    poses, K = _ring_cams(n_views, H, W)
    if kind[0] == "plane":          # views from the side the normal points to
        nrm = np.asarray(kind[1])
        keep = [b for b in range(n_views) if (-(poses[b, :, :3].T @ poses[b, :, 3])) @ nrm > kind[2] + 0.5]
        poses, K = poses[keep], K[keep]
    vol = tsdf.TSDFVolume(res=res)
    p, k = _cuda(poses, K)
    o, d = ops.raygen(p, k, W, ray_idx=torch.arange(H * W, device="cuda"))
    depth = _depth_of(kind, o, d).view(-1, H, W).contiguous()
    rgb = None if rgb_fn is None else rgb_fn(depth.shape)
    tsdf.integrate_(vol, depth, p, k, rgb=rgb)
    return vol


SPHERE = ("sphere", (0.1, -0.05, 0.07), 0.6)
PLANE = ("plane", tuple(np.array([0.3, 1.0, 0.2]) / np.linalg.norm([0.3, 1.0, 0.2])), 0.1)


@pytest.mark.parametrize("kind", [SPHERE, PLANE], ids=["sphere", "plane"])
def test_analytic_surfaces(kind):
    """every vertex within one voxel of the surface; the sphere's face normals point away from its centre (>= 99 %);
    constant colour maps give exactly that colour at every vertex"""
    from sparf_b200 import tsdf
    colour = torch.tensor([0.25, 0.625, 0.8], device="cuda")
    vol = _fuse_analytic(kind, rgb_fn=lambda s: colour.expand(*s, 3).contiguous())
    m = tsdf.extract_mesh(vol)
    v, f, c = m["vertices"].double(), m["faces"], m["colors"]
    h = 2.4 / vol.res
    print("%s: V %d, F %d" % (kind[0], v.shape[0], f.shape[0]))
    assert f.shape[0] > 1000
    assert f.min().item() >= 0 and f.max().item() < v.shape[0]
    if kind[0] == "sphere":
        ctr = torch.tensor(kind[1], dtype=torch.float64, device="cuda")
        dist = ((v - ctr).norm(dim=-1) - kind[2]).abs()
        fn = torch.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]], dim=-1)
        out = ((fn * (v[f].mean(1) - ctr)).sum(-1) > 0).double().mean().item()
        print("sphere: outward faces %.5f" % out)
        assert out >= 0.99
    else:
        nrm = torch.tensor(kind[1], dtype=torch.float64, device="cuda")
        dist = ((v * nrm).sum(-1) - kind[2]).abs()
    print("max distance to the surface %.3g voxels" % (dist.max().item() / h))
    assert dist.max().item() <= h
    assert torch.equal(c, colour.expand_as(c))


def test_linear_colour_field():
    """a colour volume linear in the lattice position gives every vertex the field's value there within 1e-5"""
    from sparf_b200 import mesh, tsdf
    vol = _fuse_analytic(SPHERE, rgb_fn=lambda s: torch.zeros(*s, 3, device="cuda"))
    A = torch.tensor([[0.2, -0.1, 0.15], [0.05, 0.3, -0.2], [-0.25, 0.1, 0.1]], device="cuda")
    b = torch.tensor([0.5, 0.45, 0.55], device="cuda")
    t = vol.axis
    pts = torch.stack(torch.meshgrid(t, t, t, indexing="ij"), -1)
    vol.color.copy_(pts @ A.T + b)
    m = tsdf.extract_mesh(vol)
    want = m["vertices"] @ A.T + b
    assert m["colors"].shape == want.shape and want.shape[0] > 1000
    assert (m["colors"] - want).abs().max().item() <= 1e-5


# ------------------------------------------------------------------------------------------------ 4. masked marching cubes
def _gaussians(shape, seed, n=6):
    rng = np.random.default_rng(seed)
    x = np.stack(np.meshgrid(*[np.arange(s, dtype=np.float64) for s in shape], indexing="ij"), -1)
    out = np.zeros(shape)
    for _ in range(n):
        c = rng.random(3) * np.array(shape)
        w = 2 + 6 * rng.random()
        out += rng.uniform(0.5, 1.5) * np.exp(-((x - c) ** 2).sum(-1) / (2 * w * w))
    return out.astype(np.float32)


def _volumes_without_nan():
    rng = np.random.default_rng(7)
    out = [(_gaussians((37, 50, 23), 0), 0.5), (_gaussians((64, 17, 40), 2), 0.6)]
    out += [(np.where(rng.random(s) < 0.5, 1.0, -1.0).astype(np.float32), 0.0) for s in ((20, 17, 31), (2, 9, 3), (33, 2, 2))]
    out += [(rng.integers(-2, 3, (19, 23, 21)).astype(np.float32), 1.0), (rng.standard_normal((15, 16, 17)).astype(np.float32), 0.3)]
    for c in range(0, 256, 5):
        vol = np.array([1.0 if c >> q & 1 else -1.0 for q in range(8)], np.float32).reshape(2, 2, 2).transpose(2, 1, 0)
        out.append((vol * np.float32(0.75) + np.float32(0.1), 0.1))
    return out


def _bits(x):
    return x.cpu().numpy().view(np.uint32) if x.dtype == torch.float32 else x.cpu().numpy()


def test_masked_is_dense_without_nan():
    from sparf_b200 import ops
    for vol, iso in _volumes_without_nan():
        x = torch.from_numpy(vol).cuda()
        a, b = ops.marching_cubes(x, iso), ops.marching_cubes_masked(x, iso)
        assert a[0].shape == b[0].shape and a[1].shape == b[1].shape
        assert np.array_equal(_bits(a[0]), _bits(b[0])) and torch.equal(a[1], b[1])


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_masked_with_nan_matches_oracle(seed):
    """NaN (and infinite) points: the dense mesh without the triangles of cells with a non-finite corner and without the
    vertices they alone used; every vertex referenced, ids in range"""
    from sparf_b200 import ops
    rng = np.random.default_rng(seed)
    vol = _gaussians((41, 38, 45), 10 + seed) if seed < 2 else rng.standard_normal((30, 31, 32)).astype(np.float32)
    bad = rng.random(vol.shape)
    vol[bad < 0.04] = np.nan
    vol[(bad >= 0.04) & (bad < 0.05)] = np.inf
    vol[(bad >= 0.05) & (bad < 0.06)] = -np.inf
    if seed == 0:
        vol[:, :, 20:] = np.nan       # a large unobserved region next to an observed one
    iso = 0.5 if seed < 2 else 0.0
    v, f = ops.marching_cubes_masked(torch.from_numpy(vol).cuda(), iso)
    rv, rf = T.masked_marching_cubes(vol, iso)
    assert v.shape == rv.shape and f.shape == rf.shape, (v.shape, rv.shape, f.shape, rf.shape)
    assert np.array_equal(_bits(v), rv.view(np.uint32)) and np.array_equal(f.cpu().numpy(), rf)
    assert len(rf) > 100 and np.isfinite(rv).all()
    used = torch.zeros(v.shape[0], dtype=torch.bool, device="cuda")
    used[f.view(-1)] = True
    assert used.all() and f.min().item() >= 0 and f.max().item() < v.shape[0]


def test_masked_count_emit_capture_and_replay():
    from sparf_b200 import _lib, ops
    L = _lib.lib()
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    shape = (41, 38, 45)
    vols = []
    for s in (20, 21):
        x = _gaussians(shape, s)
        x[np.random.default_rng(s).random(shape) < 0.03] = np.nan
        vols.append(torch.from_numpy(x).cuda())
    vol = vols[0].clone()
    iso = 0.5
    ref = [ops.marching_cubes_masked(x, iso) for x in vols]
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
        _lib.check(L.sparf_mcubes_count_masked(p(vol), *shape, iso, p(totals), p(ws), ws.numel(), st), "count_masked")
        _lib.check(L.sparf_mcubes_emit_masked(p(vol), *shape, iso, p(verts), p(faces), p(ws), ws.numel(), st), "emit_masked")
    for x, (rv, rf) in zip(vols + vols[:1], ref + ref[:1]):
        vol.copy_(x)
        graph.replay()
        torch.cuda.synchronize()
        V, F = totals.tolist()
        assert (V, F) == (rv.shape[0], rf.shape[0])
        assert torch.equal(verts[:V].view(torch.int32), rv.view(torch.int32)) and torch.equal(faces[:F], rf)


# ------------------------------------------------------------------------------------------------ 5. renders of a Graph
def _graph_scene(B=3, H=20, W=28):
    import common
    from sparf_b200.renderer import Graph
    opt = common.make_opt(S=48, S_fine=48, fine=True, depth_range=(1.5, 4.5))
    graph = Graph(opt, torch.device("cuda"))
    for i, m in enumerate(graph.get_network_components()):
        m.load_state_dict(common.det_weights(opt, 40 + i, peaky=True, sigma_bias=-2.0), strict=False)
    data = common.make_scene(3, B, H, W, focal=float(max(H, W)) * 1.3)
    return graph, opt, data.pose.cuda(), data.intr.cuda(), H, W


@pytest.mark.parametrize("config", ["dense", "grid", "termination", "grid_termination"])
def test_fuse_renders_is_integrate_of_the_val_outputs(config):
    """fuse_renders, in two batches of views, equals integrate_ of the depth / opacity, rgb and opacity >= min_opacity
    of the fine pass of one val render of all views, bit for bit, with and without an occupancy grid and early
    termination"""
    from sparf_b200 import occupancy, tsdf
    from sparf_b200.utils.edict import edict
    graph, opt, pose, intr, H, W = _graph_scene()
    with torch.no_grad():
        if "grid" in config:
            graph.set_occupancy(*[occupancy.build_grid(opt, m, res=64) for m in graph.get_network_components()])
        if "termination" in config:
            graph.set_early_termination(1e-4, 8)
        data = edict(depth_range=torch.tensor([[1.5, 4.5]], device="cuda"))
        pred = graph.render_image_at_specific_pose_and_rays(opt, data, pose, intr, H, W, iter=None, mode="val")
    opacity = pred["opacity_fine"][..., 0]
    min_opacity = opacity.median().item()           # about half of the pixels valid
    depth = (pred["depth_fine"][..., 0] / opacity).view(-1, H, W)
    ref = tsdf.TSDFVolume(res=40)
    tsdf.integrate_(ref, depth.contiguous(), pose, intr, rgb=pred["rgb_fine"].reshape(-1, H, W, 3).contiguous(),
                    valid=(opacity >= min_opacity).view(-1, H, W).contiguous())
    old = tsdf.BATCH_PIXELS
    tsdf.BATCH_PIXELS = 2 * H * W          # two batches: views (0, 1) and (2,)
    try:
        vol = tsdf.fuse_renders(opt, graph, tsdf.TSDFVolume(res=40), pose, intr, H, W, (1.5, 4.5),
                                min_opacity=min_opacity)
    finally:
        tsdf.BATCH_PIXELS = old
    assert ref.weight.sum().item() > 0
    for a in ("tsdf", "weight", "color"):
        assert torch.equal(getattr(vol, a), getattr(ref, a)), a


# ------------------------------------------------------------------------------------------------ 6. capture
def test_integrate_capture_and_replay():
    from sparf_b200 import tsdf
    B, H, W = 5, 24, 32
    poses, K = _cams(B, H, W, seed=8)
    depth, rgb, valid = _random_maps(B, H, W, seed=9)
    d, p, k, c, v = _cuda(depth, poses, K, rgb, valid)
    eager = tsdf.TSDFVolume(res=36)
    tsdf.integrate_(eager, d, p, k, rgb=c, valid=v)
    tsdf.integrate_(eager, d, p, k, rgb=c, valid=v)
    vol = tsdf.TSDFVolume(res=36)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=s):
        tsdf.integrate_(vol, d, p, k, rgb=c, valid=v)
    torch.cuda.synchronize()
    vol.reset_()
    graph.replay()
    graph.replay()
    torch.cuda.synchronize()
    for a in ("tsdf", "weight", "color"):
        assert torch.equal(getattr(vol, a), getattr(eager, a)), a


# ------------------------------------------------------------------------------------------------ 7. the tool
def test_extract_mesh_tool_tsdf(tmp_path):
    """tools/extract_mesh.py --tsdf on a snapshot and a camera file writes the PLY of tsdf.extract_mesh + write_ply"""
    import common
    from sparf_b200 import mesh, tsdf
    from sparf_b200.renderer import Graph
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import extract_mesh as tool
    from time_occupancy import octahedron_weights
    opt = common.make_opt(fine=True, depth_range=(1.5, 4.5))
    graph = Graph(opt, torch.device("cuda"))
    for i, m in enumerate(graph.get_network_components()):
        m.load_state_dict(octahedron_weights(opt, c=24.0, k=40.0, seed=i))
    ckpt = str(tmp_path / "model.pth.tar")
    torch.save({"state_dict": graph.state_dict()}, ckpt)
    B, H, W = 6, 24, 32
    poses, K = _ring_cams(B, H, W)
    cams = str(tmp_path / "cams.npz")
    np.savez(cams, pose_w2c=poses, intr=K, H=H, W=W, depth_range=np.array([1.5, 4.5], np.float32))
    out = str(tmp_path / "tool.ply")
    tool.main([ckpt, "--tsdf", cams, "--res", "48", "--trunc", "0.15", "--out", out])
    vol = tsdf.TSDFVolume(res=48, trunc=0.15)
    tsdf.fuse_renders(opt, graph, vol, torch.from_numpy(poses), torch.from_numpy(K), H, W, (1.5, 4.5))
    m = tsdf.extract_mesh(vol)
    ref = str(tmp_path / "ref.ply")
    mesh.write_ply(ref, m["vertices"], m["faces"], colors=m["colors"])
    assert m["faces"].shape[0] > 100
    with open(out, "rb") as a, open(ref, "rb") as b:
        assert a.read() == b.read()
    header, vert, _ = T.read_ply(out)
    assert "property uchar red" in header
