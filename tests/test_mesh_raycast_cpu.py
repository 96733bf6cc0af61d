"""CPU checks of the mesh ray cast: the fp64 oracle against an independent Moller-Trumbore brute force and analytic
spheres, its watertightness on shared edges, argument checks that fail before any library call, the C entry's
refusals, the binding, and the tools' new arguments."""
import ctypes
import math
import os
import sys

import numpy as np
import pytest
import torch

import raycast_oracle as RO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INVALID = 1     # SPARF_ERR_INVALID


def _icosphere(level=2):
    """a closed unit sphere: the subdivided icosahedron (vertices on the sphere)"""
    t = (1 + 5 ** 0.5) / 2
    v = [(-1, t, 0), (1, t, 0), (-1, -t, 0), (1, -t, 0), (0, -1, t), (0, 1, t), (0, -1, -t), (0, 1, -t), (t, 0, -1),
         (t, 0, 1), (-t, 0, -1), (-t, 0, 1)]
    f = [(0, 11, 5), (0, 5, 1), (0, 1, 7), (0, 7, 10), (0, 10, 11), (1, 5, 9), (5, 11, 4), (11, 10, 2), (10, 7, 6),
         (7, 1, 8), (3, 9, 4), (3, 4, 2), (3, 2, 6), (3, 6, 8), (3, 8, 9), (4, 9, 5), (2, 4, 11), (6, 2, 10), (8, 6, 7),
         (9, 8, 1)]
    v = [np.asarray(p, np.float64) / np.linalg.norm(p) for p in v]
    for _ in range(level):
        mid, nf = {}, []

        def m(a, b):
            key = (min(a, b), max(a, b))
            if key not in mid:
                p = v[a] + v[b]
                v.append(p / np.linalg.norm(p))
                mid[key] = len(v) - 1
            return mid[key]
        for a, b, c in f:
            ab, bc, ca = m(a, b), m(b, c), m(c, a)
            nf += [(a, ab, ca), (b, bc, ab), (c, ca, bc), (ab, bc, ca)]
        f = nf
    return np.asarray(v, np.float32).astype(np.float64), np.asarray(f, np.int64)


def test_oracle_matches_moller_trumbore():
    rng = np.random.default_rng(0)
    v = rng.normal(size=(300, 3))
    f = rng.integers(0, 300, (200, 3))
    o = rng.normal(size=(2000, 3)) * 3
    d = rng.normal(size=(2000, 3))
    t, face, bary = RO.raycast(o, d, v, f)
    tm, fm = RO.moller_trumbore(o, d, v, f)
    assert (face >= 0).sum() > 200
    assert np.array_equal(face >= 0, fm >= 0)
    h = face >= 0
    assert np.allclose(t[h], tm[h], rtol=1e-9, atol=1e-9) and np.array_equal(face[h], fm[h])
    p = o[h] + t[h, None] * d[h]
    assert np.allclose((bary[h, :, None] * v[f[face[h]]]).sum(1), p, atol=1e-9)
    assert np.allclose(bary[h].sum(1), 1) and (bary[h] >= 0).all()


def test_oracle_on_an_analytic_sphere():
    v, f = _icosphere(4)
    rng = np.random.default_rng(1)
    o = rng.normal(size=(3000, 3))
    o = 4 * o / np.linalg.norm(o, axis=1, keepdims=True)
    d = rng.uniform(-0.8, 0.8, (3000, 3)) - o
    t, face, _ = RO.raycast(o, d, v, f)
    A, B, C = (d * d).sum(1), 2 * (o * d).sum(1), (o * o).sum(1) - 1
    disc = B * B - 4 * A * C
    closest = np.linalg.norm(o - ((o * d).sum(1) / A)[:, None] * d, axis=1)
    inner = math.cos(math.radians(6.0))     # every face lies between this radius and the sphere (edges < 6 degrees)
    assert (face[closest < inner] >= 0).all() and (face[closest > 1] < 0).all()
    h = face >= 0
    t_an = (-B - np.sqrt(np.maximum(disc, 0))) / (2 * A)
    r = np.linalg.norm(o[h] + t[h, None] * d[h], axis=1)
    assert (r >= inner).all() and (r <= 1 + 1e-9).all() and (t[h] >= t_an[h] - 1e-9).all()
    # from the centre every ray hits
    t, face, _ = RO.raycast(np.zeros((2000, 3)), rng.normal(size=(2000, 3)), v, f)
    assert (face >= 0).all()


def test_oracle_is_watertight_on_shared_edges():
    """rays from inside a closed sphere aimed exactly at every vertex and edge midpoint all hit"""
    v, f = _icosphere(2)
    e = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
    targets = np.concatenate([v, (v[e[:, 0]] + v[e[:, 1]]) / 2])
    for o in (np.zeros(3), np.array([0.11, -0.23, 0.05])):
        _, face, _ = RO.raycast(np.broadcast_to(o, targets.shape), targets - o, v, f)
        assert (face >= 0).all()
    # a ray exactly through a shared edge of two coplanar triangles hits one of them
    vq = np.array([[0, 0, 0], [1, 0, 0], [1, 1, 0], [0, 1, 0]], np.float64)
    fq = np.array([[0, 1, 2], [0, 2, 3]])
    s = np.linspace(0.05, 0.95, 19)
    o = np.stack([s, s, np.full_like(s, 1.0)], 1)
    _, face, _ = RO.raycast(o, np.tile([0.0, 0.0, -1.0], (len(s), 1)), vq, fq)
    assert (face == 0).all()        # both hit at the same t: the smaller id


def test_oracle_misses_and_degenerate_faces():
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [2, 2, 0], [3, 3, 0]], np.float64)
    f = np.array([[0, 3, 4], [1, 1, 2], [0, 1, 2], [0, 1, 9]])        # collinear, repeated id, a triangle, a bad id
    o = np.array([[0.2, 0.2, 1], [2.5, 2.5, 1], [np.nan, 0, 1], [0.2, 0.2, 1], [0.2, 0.2, 1], [5, 5, 1]])
    d = np.array([[0, 0, -1], [0, 0, -1], [0, 0, -1], [0, 0, 0], [0, 0, 1], [0, 0, -1]], np.float64)
    t, face, bary = RO.raycast(o, d, v, f)
    assert face.tolist() == [2, -1, -1, -1, -1, -1]
    assert t[0] == 1.0 and np.isinf(t[1:]).all() and np.isnan(bary[1:]).all()
    t, face, _ = RO.raycast(o[:1], d[:1], v, f, t_min=1.5)
    assert face.tolist() == [-1]


# ------------------------------------------------------------------------------------------------ argument checks
def _no_library_call(monkeypatch):
    from sparf_b200 import _lib

    def refuse():
        raise AssertionError("the library was called")
    monkeypatch.setattr(_lib, "lib", refuse)


def test_raycast_rejects_bad_arguments(monkeypatch):
    from sparf_b200 import ops
    _no_library_call(monkeypatch)
    v = torch.zeros(5, 3, device="meta")
    f = torch.zeros(4, 3, dtype=torch.int64, device="meta")
    g = ops.DistanceGrid(v, f, None, None, None, (1, 1, 1), 0)
    points = ops.DistanceGrid(v, None, None, None, None, (1, 1, 1), 0)
    o = torch.zeros(7, 3, device="meta")
    inf, nan = float("inf"), float("nan")
    for args in [(None, o, o), (points, o, o), (g, o.double(), o), (g, o, o[:, :2]), (g, o[0], o), (g, o, o[:6]),
                 (g, torch.zeros(7, 3), o), (g, o, torch.zeros(7, 3)), (g, o, o, -1.0), (g, o, o, 2.0, 1.0),
                 (g, o, o, nan), (g, o, o, 0.0, nan), (g, o, o, "0"), (g, o, o, True)]:
        with pytest.raises(ValueError):
            ops.raycast(*args)


def test_render_cull_reject_bad_arguments(monkeypatch):
    from sparf_b200 import mesh
    _no_library_call(monkeypatch)
    dev = "meta"
    m = dict(vertices=torch.zeros(5, 3, device=dev), faces=torch.zeros(4, 3, dtype=torch.int64, device=dev))
    pose = torch.zeros(2, 3, 4, device=dev)
    K = torch.zeros(3, 3, device=dev)
    bad = [dict(m=dict(vertices=m["vertices"])), dict(pose=pose[0]), dict(pose=pose.double()), dict(pose=pose[:0]),
           dict(K=K[:2]), dict(K=torch.zeros(3, 3, 3, device=dev)), dict(K=K.double()), dict(H=0), dict(W=1.5),
           dict(H=True), dict(masks=torch.zeros(2, 4, 5, device=dev)), dict(masks=torch.zeros(2, 5, 4, dtype=torch.bool,
                                                                                                device=dev)),
           dict(pose=torch.zeros(2, 3, 4)), dict(K=torch.zeros(3, 3))]
    for b in bad:
        kw = dict(dict(m=m, pose=pose, K=K, H=4, W=5, masks=None), **b)
        for fn in (mesh.visible_faces, mesh.cull):
            with pytest.raises(ValueError):
                fn(kw["m"], kw["pose"], kw["K"], kw["H"], kw["W"], masks=kw["masks"])
        if b.get("masks") is None:
            with pytest.raises(ValueError):
                mesh.render(kw["m"], kw["pose"], kw["K"], kw["H"], kw["W"])
    for near, far in ((-1.0, 2.0), (2.0, 1.0), (float("nan"), 1.0), (0.0, float("nan"))):
        with pytest.raises(ValueError):
            mesh.render(m, pose, K, 4, 5, near=near, far=far)
    with pytest.raises(ValueError):
        mesh.render(m, pose, K, 4, 5, grid="grid")
    with pytest.raises(ValueError):       # a CPU mesh: there is no CPU path
        mesh.render({k: torch.zeros(v.shape, dtype=v.dtype) for k, v in m.items()}, torch.zeros(2, 3, 4),
                    torch.zeros(3, 3), 4, 5)


# ------------------------------------------------------------------------------------------------ C entry, binding
def test_declared_and_bound():
    from sparf_b200 import _lib
    src = open(os.path.join(ROOT, "include", "sparf_b200.h")).read()
    assert "sparf_raycast(" in src and "sparf_raycast" in _lib.exported_symbols()
    assert hasattr(_lib.lib(), "sparf_raycast")


def test_c_entry_point_rejects_invalid_arguments():
    """SPARF_ERR_INVALID before anything is read or launched (the pointers are host dummies)"""
    from sparf_b200 import _lib
    L = _lib.lib()
    buf = (ctypes.c_int64 * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    def cast(V=5, F=3, N=1, t0=0.0, t1=1.0, null=()):
        q = lambda name: None if name in null else p
        return L.sparf_raycast(q("v"), V, q("f"), F, q("g"), q("cs"), p, q("o"), q("d"), N, t0, t1, q("t"), q("face"),
                               q("bary"), None)
    for V, F in ((-1, 0), (1 << 31, 0), (5, -1), (5, 1 << 31), (0, 1)):
        assert cast(V=V, F=F) == INVALID, (V, F)
        assert L.sparf_last_error()
    for N in (-1, 1 << 31):
        assert cast(N=N) == INVALID, N
    nan, inf = float("nan"), float("inf")
    for t0, t1 in ((-1.0, 1.0), (2.0, 1.0), (nan, 1.0), (0.0, nan), (inf, 1.0)):
        assert cast(t0=t0, t1=t1) == INVALID, (t0, t1)
    for null in ("o", "d", "t", "face", "bary", "v", "f", "g", "cs"):
        assert cast(null=(null,)) == INVALID, null


# ------------------------------------------------------------------------------------------------ the tools
def _tools():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import compare_mesh
    import extract_mesh
    return compare_mesh, extract_mesh


def test_tool_arguments_parse():
    compare_mesh, extract_mesh = _tools()
    a = compare_mesh.parse_args(compare_mesh.build_parser(), ["p.ply", "r.ply", "--threshold", "0.01"])
    assert a.cull is None
    a = compare_mesh.parse_args(compare_mesh.build_parser(), ["p.ply", "r.ply", "--threshold", "0.01", "--cull",
                                                              "cams.npz"])
    assert a.cull == "cams.npz"
    a = extract_mesh.parse_args(extract_mesh.build_parser(), ["m.pth", "--out", "o.ply"])
    assert a.cull is None
    a = extract_mesh.parse_args(extract_mesh.build_parser(), ["m.pth", "--out", "o.ply", "--cull", "c.pt",
                                                              "--keep-largest", "1", "--simplify", "100"])
    assert (a.cull, a.keep_largest, a.simplify) == ("c.pt", 1, 100)


def test_camera_files_with_and_without_mask_and_depth_range(tmp_path):
    _, extract_mesh = _tools()
    pose = np.zeros((2, 3, 4), np.float32)
    pose[:, :, :3] = np.eye(3)
    K = np.tile(np.eye(3, dtype=np.float32), (2, 1, 1))
    mask = np.zeros((2, 4, 5), bool)
    mask[1, 2, 3] = True
    np.savez(tmp_path / "a.npz", pose_w2c=pose, intr=K, H=4, W=5, depth_range=np.array([1.0, 3.0]))
    np.savez(tmp_path / "b.npz", pose_w2c=pose, intr=K, H=4, W=5, mask=mask.astype(np.uint8))
    torch.save(dict(pose_w2c=torch.from_numpy(pose), intr=torch.from_numpy(K), H=4, W=5, mask=torch.from_numpy(mask)),
               tmp_path / "c.pt")
    p, k, H, W, dr, m = extract_mesh.load_cameras(str(tmp_path / "a.npz"))
    assert p.shape == (2, 3, 4) and k.dtype == torch.float32 and (H, W) == (4, 5) and dr == (1.0, 3.0) and m is None
    for name in ("b.npz", "c.pt"):
        p, k, H, W, dr, m = extract_mesh.load_cameras(str(tmp_path / name))
        assert dr is None and m.dtype == torch.bool and torch.equal(m, torch.from_numpy(mask))
