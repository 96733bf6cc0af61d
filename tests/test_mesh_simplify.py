"""GPU tests of the mesh simplification (csrc/mesh_simplify.cu): bytes equal to the NumPy oracle
(tests/simplify_oracle.py) on marching-cubes spheres and tori, an open grid and a soup; the invariants at a million
faces; flat grids; attributes; determinism; edge cases; the three extractors; CUDA-graph capture; the tool."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

import mcubes_oracle as O
import simplify_oracle as SO
import test_mesh_components as TMC

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _mc(vol):
    from sparf_b200 import ops
    return ops.marching_cubes(torch.from_numpy(np.ascontiguousarray(vol, np.float32)).cuda(), 0.0)


def _sphere(n, r):
    return _mc(TMC._ball((n,) * 3, ((n - 1) / 2 + 0.13,) * 3, r))


def _torus(n, R, r):
    c = (n - 1) / 2 + 0.11
    return _mc(TMC._torus((n,) * 3, (c, c, c), R, r))


def _grid(n, jitter=0.2, flat=False, seed=0):
    """an open n x n vertex grid, two triangles per cell"""
    rng = np.random.default_rng(seed)
    g = np.stack(np.meshgrid(np.arange(n), np.arange(n), indexing="ij"), -1).reshape(-1, 2).astype(np.float32)
    g += rng.uniform(-jitter, jitter, g.shape).astype(np.float32)
    z = np.zeros((len(g), 1), np.float32) if flat else rng.uniform(-0.3, 0.3, (len(g), 1)).astype(np.float32)
    a = (np.arange(n - 1)[:, None] * n + np.arange(n - 1)[None, :]).reshape(-1)
    f = np.stack([np.stack([a, a + n, a + 1], 1), np.stack([a + 1, a + n, a + n + 1], 1)], 1).reshape(-1, 3)
    return torch.from_numpy(np.concatenate([g, z], 1)).cuda(), torch.from_numpy(f.astype(np.int64)).cuda()


def _soup():
    """a jittered grid plus a fin on a non-manifold edge, degenerate faces and unused vertices"""
    v, f = _grid(12, seed=3)
    V = v.shape[0]
    extra_v = torch.tensor([[5.0, 5.0, 3.0], [40.0, 40.0, 40.0], [41.0, 40.0, 40.0]], device="cuda")
    extra_f = torch.tensor([[13, 14, V], [20, 20, 33], [50, 51, 50]], dtype=torch.int64, device="cuda")
    return torch.cat([v, extra_v]), torch.cat([f, extra_f])


MESHES = {"sphere": lambda: _sphere(14, 4.3), "torus": lambda: _torus(18, 5.0, 2.2), "grid": lambda: _grid(16),
          "soup": _soup}


def _attrs(v):
    g = torch.Generator(device="cpu").manual_seed(0)
    return torch.rand(v.shape[0], 4, generator=g).cuda()


def _check_oracle(v, f, target, attrs=None):
    from sparf_b200 import ops
    st = {}
    got = ops.mesh_simplify(v, f, target, attrs=attrs, stats=st)
    ref = SO.simplify(v.cpu().numpy(), f.cpu().numpy(), target, None if attrs is None else attrs.cpu().numpy())
    for g, r in zip(got, ref[:4]):
        assert (g is None) == (r is None)
        if g is not None:
            assert torch.equal(g.cpu(), torch.from_numpy(np.asarray(r)).reshape(g.shape)), (g.shape, r.shape)
    assert st["rounds"] == ref[4]
    return got, st


@pytest.mark.parametrize("name", sorted(MESHES))
@pytest.mark.parametrize("frac", [0.0, 0.1, 0.5, 1.0, 1.5])
def test_matches_oracle(name, frac):
    v, f = MESHES[name]()
    assert 200 < f.shape[0] < 2000
    target = int(frac * f.shape[0]) + (1 if frac > 1 else 0)
    (vo, fo, ids, ao), st = _check_oracle(v, f, target, attrs=_attrs(v) if name != "grid" else None)
    if target >= f.shape[0]:
        assert st["rounds"] == 0 and torch.equal(vo, v) and torch.equal(fo, f)
    elif name in ("sphere", "torus") and frac > 0:
        assert fo.shape[0] <= target


# ------------------------------------------------------------------------------------------------ invariants at scale
def _euler(f, V):
    e = np.unique(np.sort(np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]]), 1), axis=0)
    return V - len(e) + len(f)


def _areas(v, f):
    p = v[f]
    return np.linalg.norm(np.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0]), axis=1)


def _volume(v, f):
    p = v[f].astype(np.float64)
    return np.einsum("ij,ij->i", p[:, 0], np.cross(p[:, 1], p[:, 2])).sum() / 6


@pytest.mark.parametrize("shape", ["sphere", "torus"])
def test_invariants_at_a_million_faces(shape):
    from sparf_b200 import ops
    if shape == "sphere":
        n, R, r = 384, 0.0, 175.0
        v, f = _sphere(n, r)
        c = (n - 1) / 2 + 0.13
    else:
        n, R, r = 448, 140.0, 70.0
        v, f = _torus(n, R, r)
        c = (n - 1) / 2 + 0.11
    F = f.shape[0]
    assert F >= 1_000_000
    target = F // 100
    st = {}
    vo, fo, ids, _ = ops.mesh_simplify(v, f, target, stats=st)
    vn, fn, vi, fi = vo.cpu().numpy(), fo.cpu().numpy(), v.cpu().numpy(), f.cpu().numpy()
    print("%s: F %d -> %d in %d rounds" % (shape, F, fn.shape[0], st["rounds"]))
    assert fn.shape[0] <= target
    assert O.is_closed_and_oriented(fn)
    assert _euler(fn, len(vn)) == _euler(fi, len(vi)) == (2 if shape == "sphere" else 0)
    assert (_areas(vn, fn) == 0).sum() <= (_areas(vi, fi) == 0).sum()
    d = vn - c
    if shape == "sphere":
        dist = np.abs(np.linalg.norm(d, axis=1) - r)
    else:
        dist = np.abs(np.hypot(np.hypot(d[:, 0], d[:, 1]) - R, d[:, 2]) - r)
    vol0, vol1 = _volume(vi, fi), _volume(vn, fn)
    print("%s: max distance %.3f voxels, volume %.5f relative" % (shape, dist.max(), vol1 / vol0 - 1))
    assert dist.max() < 0.5
    assert abs(vol1 / vol0 - 1) < 2e-3


def test_flat_open_grid():
    from sparf_b200 import ops
    v, f = _grid(101, jitter=0.3, flat=True)
    vo, fo, ids, _ = ops.mesh_simplify(v, f, 200)
    n = 101
    i, j = np.divmod(np.arange(n * n), n)
    border = np.flatnonzero((i == 0) | (j == 0) | (i == n - 1) | (j == n - 1))
    ids = ids.cpu().numpy()
    assert np.isin(border, ids).all()
    pos = dict(zip(ids.tolist(), range(len(ids))))
    assert vo.cpu().numpy()[[pos[b] for b in border]].tobytes() == v.cpu().numpy()[border].tobytes()
    assert (vo[:, 2] == 0).all()
    assert _euler(fo.cpu().numpy(), vo.shape[0]) == 1 and fo.shape[0] < f.shape[0] // 10


def test_attributes():
    from sparf_b200 import mesh
    v, f = _sphere(64, 25.0)
    colors = torch.rand(v.shape[0], 3, device="cuda")
    colors[:, 1] = 0.375
    normals = torch.nn.functional.normalize(v - v.mean(0), dim=1)
    st = {}
    m = mesh.simplify(dict(vertices=v, faces=f, colors=colors, normals=normals, tag="x"), f.shape[0] // 20, stats=st)
    assert st["reached"] and st["faces_after"] == m["faces"].shape[0] <= f.shape[0] // 20 and m["tag"] == "x"
    c = m["colors"]
    assert (c[:, 1] == 0.375).all()
    for ch in (0, 2):
        assert c[:, ch].min() >= colors[:, ch].min() and c[:, ch].max() <= colors[:, ch].max()
    ln = m["normals"].norm(dim=1)
    assert ((ln - 1).abs() < 1e-6).logical_or(ln == 0).all()


def _parametric_torus(nu, nv, R=3.0, r=1.0):
    u = torch.arange(nu, device="cuda", dtype=torch.float64) * (2 * np.pi / nu)
    w = torch.arange(nv, device="cuda", dtype=torch.float64) * (2 * np.pi / nv)
    U, W = torch.meshgrid(u, w, indexing="ij")
    x = torch.stack([(R + r * W.cos()) * U.cos(), (R + r * W.cos()) * U.sin(), r * W.sin()], -1).reshape(-1, 3)
    i, j = torch.meshgrid(torch.arange(nu, device="cuda"), torch.arange(nv, device="cuda"), indexing="ij")
    a, b = i * nv + j, ((i + 1) % nu) * nv + j
    c, d = i * nv + (j + 1) % nv, ((i + 1) % nu) * nv + (j + 1) % nv
    f = torch.stack([torch.stack([a, b, c], -1), torch.stack([c, b, d], -1)], -2).reshape(-1, 3)
    return x.float().contiguous(), f.contiguous()


def test_determinism_at_ten_million_faces():
    from sparf_b200 import ops
    v, f = _parametric_torus(2500, 2000)
    assert f.shape[0] >= 10_000_000
    a = ops.mesh_simplify(v, f, f.shape[0] // 10)
    b = ops.mesh_simplify(v, f, f.shape[0] // 10)
    for x, y in zip(a[:3], b[:3]):
        assert x.cpu().numpy().tobytes() == y.cpu().numpy().tobytes()
    assert a[1].shape[0] <= f.shape[0] // 10


def test_edge_cases():
    from sparf_b200 import ops
    v, f = _sphere(14, 4.3)
    for t in (f.shape[0], f.shape[0] + 5):
        vo, fo, ids, ao = ops.mesh_simplify(v, f, t, attrs=_attrs(v))
        assert torch.equal(vo, v) and torch.equal(fo, f) and torch.equal(ids, torch.arange(v.shape[0], device="cuda"))
        assert torch.equal(ao, _attrs(v))
    e = torch.zeros(0, 3, dtype=torch.int64, device="cuda")
    vo, fo, ids, ao = ops.mesh_simplify(torch.zeros(0, 3, device="cuda"), e, 0)
    assert vo.shape == (0, 3) and fo.shape == (0, 3) and ids.shape == (0,) and ao is None
    vo, fo, ids, _ = ops.mesh_simplify(v, e, 0)
    assert torch.equal(vo, v) and fo.shape == (0, 3)


# ------------------------------------------------------------------------------------------------ the extractors
def _check_manifold_components(m0, m1):
    from sparf_b200 import ops
    def chis(m):
        f, V = m["faces"], m["vertices"].shape[0]
        labels, counts = ops.mesh_components(f, V)
        lab = labels.cpu().numpy()[f[:, 0].cpu().numpy()]
        fn = f.cpu().numpy()
        return sorted(_euler(fn[lab == c], len(np.unique(fn[lab == c]))) for c in range(counts.numel())
                      if counts[c] > 0)
    fn = m1["faces"].cpu().numpy()
    e = np.sort(np.concatenate([fn[:, [0, 1]], fn[:, [1, 2]], fn[:, [2, 0]]]), 1)
    _, cnt = np.unique(e, axis=0, return_counts=True)
    assert cnt.max() <= 2
    assert chis(m0) == chis(m1)


@pytest.mark.parametrize("sparse", [False, True])
def test_extractors(sparse):
    from sparf_b200 import mesh
    opt, (_, blobs) = TMC._nerfs(res=128)
    m = (mesh.extract_mesh_sparse if sparse else mesh.extract_mesh)(opt, blobs, normals=True)
    st = {}
    got = mesh.simplify(m, m["faces"].shape[0] // 10, stats=st)
    print("extractor: %s" % st)
    assert st["reached"]
    _check_manifold_components(m, got)


def test_tsdf_mesh():
    import common
    from sparf_b200 import mesh, tsdf
    from sparf_b200.renderer import Graph
    opt = common.make_opt(fine=True, depth_range=(1.5, 4.5))
    graph = Graph(opt, torch.device("cuda"))
    for i, net in enumerate(graph.get_network_components()):
        net.load_state_dict({k: v.cuda() for k, v in
                             TMC.blob_weights(opt, [TMC.MAIN_TSDF] + TMC.BLOBS_TSDF, seed=i).items()})
    poses, Kc = TMC._ring_cams(12, 60, 80)
    vol = tsdf.TSDFVolume(res=64)
    tsdf.fuse_renders(opt, graph, vol, torch.from_numpy(poses), torch.from_numpy(Kc), 60, 80, (1.5, 4.5))
    m = tsdf.extract_mesh(vol)
    got = mesh.simplify(m, m["faces"].shape[0] // 4)
    assert got["colors"].shape == (got["vertices"].shape[0], 3)
    _check_manifold_components(m, got)
    # the open border of the observed surface stays where it was
    fn = m["faces"].cpu().numpy()
    e = np.sort(np.concatenate([fn[:, [0, 1]], fn[:, [1, 2]], fn[:, [2, 0]]]), 1)
    u, cnt = np.unique(e, axis=0, return_counts=True)
    border = np.unique(u[cnt == 1])
    v0 = m["vertices"].cpu().numpy()
    kept = {tuple(p) for p in got["vertices"].cpu().numpy().tolist()}
    assert all(tuple(p) in kept for p in v0[border].tolist())


# ------------------------------------------------------------------------------------------------ capture
def test_capture_round_replays_eager_bytes():
    """one round captured in a CUDA graph: each replay (after a fresh init) emits the eager round's bytes"""
    from sparf_b200 import _lib
    L = _lib.lib()
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    st = lambda: ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    v, f = _sphere(40, 15.0)
    a = _attrs(v)
    V, F, A = v.shape[0], f.shape[0], a.shape[1]
    ws = torch.zeros(L.sparf_mesh_simplify_workspace_bytes(V, F, A), dtype=torch.uint8, device="cuda")
    counts = torch.zeros(2, dtype=torch.int64, device="cuda")
    k = F // 4

    def init():
        _lib.check(L.sparf_mesh_simplify_init(p(v), p(f), p(a), V, F, A, p(counts), p(ws), ws.numel(), st()), "init")

    def emit():
        torch.cuda.synchronize()
        n, won = counts.tolist()
        out = (torch.empty(V - won, 3, device="cuda"), torch.empty(V - won, A, device="cuda"),
               torch.empty(V - won, dtype=torch.int64, device="cuda"), torch.empty(n, 3, dtype=torch.int64, device="cuda"))
        _lib.check(L.sparf_mesh_simplify_emit(V, F, A, n, *[p(t) for t in out], p(ws), ws.numel(), st()), "emit")
        torch.cuda.synchronize()
        return counts.clone(), out

    init()
    _lib.check(L.sparf_mesh_simplify_round(V, F, A, F, k, p(counts), p(ws), ws.numel(), st()), "round")
    ref_counts, ref = emit()
    assert ref_counts[1] > 0 and O.is_closed_and_oriented(ref[3].cpu().numpy())
    init()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        _lib.check(L.sparf_mesh_simplify_round(V, F, A, F, k, p(counts), p(ws), ws.numel(), st()), "round")
    for _ in range(2):
        init()
        g.replay()
        got_counts, got = emit()
        assert torch.equal(got_counts, ref_counts) and all(torch.equal(x, y) for x, y in zip(got, ref))


# ------------------------------------------------------------------------------------------------ the tool
def test_extract_mesh_tool_simplify(tmp_path):
    """tools/extract_mesh.py --simplify F writes the bytes of mesh.simplify + write_ply (normals at the final vertices)"""
    from sparf_b200 import mesh
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import extract_mesh as tool
    opt, (_, blobs) = TMC._nerfs(res=64)
    ckpt = str(tmp_path / "model.pth.tar")
    torch.save({"state_dict": {"nerf." + k: v for k, v in blobs.state_dict().items()}}, ckpt)
    for extra, extract in (([], mesh.extract_mesh), (["--sparse"], mesh.extract_mesh_sparse)):
        out = str(tmp_path / "tool.ply")
        tool.main([ckpt, "--res", "64", "--thres", str(TMC.ISO), "--normals", "--keep-largest", "1", "--simplify",
                   "1000", "--out", out] + extra)
        m = mesh.simplify(mesh.keep_components(extract(opt, blobs), largest=1), 1000)
        n = mesh.density_normals(blobs, m["vertices"])
        ref = str(tmp_path / "ref.ply")
        mesh.write_ply(ref, m["vertices"], m["faces"], n)
        assert 0 < m["faces"].shape[0] <= 1000
        with open(out, "rb") as a, open(ref, "rb") as b:
            assert a.read() == b.read()
