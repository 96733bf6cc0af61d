"""CPU checks of the mesh distance: the fp64 oracle's own correctness, read_ply against write_ply and hand-written
files, the metric formulas, argument checks that fail before any library call, the C entries' refusals, the bindings,
and the tool's arguments."""
import ctypes
import math
import os
import sys

import numpy as np
import pytest
import torch

import mesh_distance_oracle as MD

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INVALID = 1     # SPARF_ERR_INVALID
ENTRY_POINTS = ["sparf_distance_grid_workspace_bytes", "sparf_distance_grid_count", "sparf_distance_grid_fill",
                "sparf_distance_query"]


# ------------------------------------------------------------------------------------------------ the oracle
def _random_triangles(n, seed=0):
    rng = np.random.default_rng(seed)
    return rng.normal(size=(n, 3)), rng.normal(size=(n, 3)), rng.normal(size=(n, 3)), rng.normal(size=(n, 3)) * 2


def test_oracle_closest_points_lie_on_their_triangles():
    a, b, c, p = _random_triangles(5000)
    q, d2 = MD.closest_on_triangle(p, a, b, c)
    w = MD.barycentric(q, a, b, c)
    assert (w > -1e-9).all() and (w < 1 + 1e-9).all()
    assert np.allclose(d2, ((p - q) ** 2).sum(1))


def test_oracle_interior_residual_is_orthogonal_to_the_face():
    a, b, c, p = _random_triangles(5000, seed=1)
    q, _ = MD.closest_on_triangle(p, a, b, c)
    w = MD.barycentric(q, a, b, c)
    interior = (w > 1e-6).all(1)
    assert interior.sum() > 200
    r = (p - q)[interior]
    for e in (b - a, c - a):
        e = e[interior]
        cos = (r * e).sum(1) / (np.linalg.norm(r, axis=1) * np.linalg.norm(e, axis=1))
        assert np.abs(cos).max() < 1e-9


def test_oracle_is_at_most_dense_sampling():
    a, b, c, p = _random_triangles(300, seed=2)
    _, d2 = MD.closest_on_triangle(p, a, b, c)
    g = np.linspace(0, 1, 41)
    u, v = np.meshgrid(g, g, indexing="ij")
    keep = (u + v) <= 1
    u, v = u[keep], v[keep]
    pts = a[:, None] + u[None, :, None] * (b - a)[:, None] + v[None, :, None] * (c - a)[:, None]
    sampled = ((pts - p[:, None]) ** 2).sum(-1).min(1)
    assert (d2 <= sampled + 1e-12).all()
    assert np.median(sampled - d2) < 1e-2      # and close to them


def test_oracle_degenerate_triangles():
    p = np.array([[0.5, 1.0, 0.0], [3.0, 0.0, 0.0], [-1.0, -1.0, 0.0]])
    seg = lambda q, a, b: MD.closest_on_segment(q, a, b)
    # repeated vertex: the segment a-c
    a, c = np.array([0.0, 0, 0]), np.array([2.0, 0, 0])
    q, d2 = MD.closest_on_triangle(p, a, a, c)
    assert np.allclose(q, seg(p, a, c)) and np.allclose(d2, [1.0, 1.0, 2.0])
    # collinear: the hull of the three points, the segment from the first to the last
    q, d2 = MD.closest_on_triangle(p, np.array([0.0, 0, 0]), np.array([1.0, 0, 0]), np.array([2.0, 0, 0]))
    assert np.allclose(d2, [1.0, 1.0, 2.0])
    # a point triangle
    q, d2 = MD.closest_on_triangle(p, a, a, a)
    assert np.allclose(q, 0) and np.allclose(d2, (p ** 2).sum(1))


def test_oracle_brute_force_ties_and_misses():
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]], np.float64)
    f = np.array([[0, 1, 2], [0, 1, 2], [0, 1, 3]])
    d, i, q = MD.closest_triangles(np.array([[0.2, 0.2, 1.0], [0.2, 0.2, -5.0]]), v, f, max_dist=2.0)
    assert i.tolist() == [2, -1] and d[0] == pytest.approx(math.sqrt(0.06))     # the edge (1,0,0)-(0,0,1) of face 2
    assert np.isinf(d[1]) and np.isnan(q[1]).all()
    d, i, _ = MD.closest_triangles(np.array([[0.2, 0.2, -0.5]]), v, f)
    assert i.tolist() == [0] and d[0] == pytest.approx(0.5)        # faces 0 and 1 tie: the smaller id
    d, i, _ = MD.closest_vertices(np.array([[0.9, 0, 0]]), v)
    assert i.tolist() == [1] and d[0] == pytest.approx(0.1)


# ------------------------------------------------------------------------------------------------ read_ply
def _mesh(V=50, F=80, seed=0):
    rng = np.random.default_rng(seed)
    return (torch.from_numpy(rng.normal(size=(V, 3)).astype(np.float32)),
            torch.from_numpy(rng.integers(0, V, (F, 3))), torch.from_numpy(rng.normal(size=(V, 3)).astype(np.float32)),
            torch.from_numpy(rng.random((V, 3)).astype(np.float32)))


@pytest.mark.parametrize("case", ["plain", "normals", "colors", "both", "empty", "points"])
def test_read_ply_round_trips_write_ply(tmp_path, case):
    from sparf_b200 import mesh
    v, f, n, c = _mesh()
    if case == "empty":
        v, f, n, c = v[:0], f[:0], None, None
    if case == "points":
        f = f[:0]
    n = n if case in ("normals", "both") else None
    c = c if case in ("colors", "both") else None
    a, b = tmp_path / "a.ply", tmp_path / "b.ply"
    mesh.write_ply(a, v, f, normals=n, colors=c)
    m = mesh.read_ply(a)
    assert torch.equal(m["vertices"], v) and torch.equal(m["faces"], f)
    assert ("normals" in m) == (n is not None) and ("colors" in m) == (c is not None)
    mesh.write_ply(b, m["vertices"], m["faces"], normals=m.get("normals"), colors=m.get("colors"))
    assert a.read_bytes() == b.read_bytes()


ASCII = """ply
format ascii 1.0
comment hand written
element vertex 4
property double x
property double y
property double z
property float confidence
property uchar red
property uchar green
property uchar blue
element face 2
property list int int vertex_indices
end_header
0 0 0 0.5 255 0 0
1 0 0 0.5 0 255 0
0 1.5 0 0.5 0 0 255
0 0 2.25 0.5 51 51 51
3 0 1 2
3 0 3 1
"""


def test_read_ply_hand_written_ascii(tmp_path):
    from sparf_b200 import mesh
    p = tmp_path / "m.ply"
    p.write_text(ASCII)
    m = mesh.read_ply(p)
    assert m["vertices"].dtype == torch.float32 and m["vertices"][2, 1] == 1.5 and m["vertices"][3, 2] == 2.25
    assert m["faces"].tolist() == [[0, 1, 2], [0, 3, 1]] and m["faces"].dtype == torch.int64
    assert torch.allclose(m["colors"][3], torch.full((3,), 0.2)) and m["colors"][0, 0] == 1.0
    assert "normals" not in m
    p.write_text(ASCII.replace("element face 2\nproperty list int int vertex_indices\n", "").rsplit("3 0 1 2", 1)[0])
    pc = mesh.read_ply(p)
    assert "faces" not in pc and pc["vertices"].shape == (4, 3)


def test_read_ply_binary_point_cloud_with_extra_properties(tmp_path):
    from sparf_b200 import mesh
    dt = np.dtype([("x", "<f8"), ("y", "<f8"), ("z", "<f8"), ("value", "<i2"), ("nx", "<f4"), ("ny", "<f4"),
                   ("nz", "<f4")])
    a = np.zeros(3, dt)
    a["x"], a["y"], a["z"], a["nz"] = [1, 2, 3], [4, 5, 6], [7, 8, 9], 1
    head = ("ply\nformat binary_little_endian 1.0\nelement vertex 3\nproperty double x\nproperty double y\n"
            "property double z\nproperty short value\nproperty float nx\nproperty float ny\nproperty float nz\n"
            "end_header\n")
    p = tmp_path / "pc.ply"
    p.write_bytes(head.encode() + a.tobytes())
    m = mesh.read_ply(p)
    assert "faces" not in m and m["vertices"][:, 0].tolist() == [1, 2, 3] and (m["normals"][:, 2] == 1).all()


def test_read_ply_rejects_big_endian_quads_and_vertex_lists(tmp_path):
    from sparf_b200 import mesh
    p = tmp_path / "x.ply"
    p.write_bytes(b"ply\nformat binary_big_endian 1.0\nelement vertex 0\nproperty float x\nproperty float y\n"
                  b"property float z\nend_header\n")
    with pytest.raises(ValueError, match="format"):
        mesh.read_ply(p)
    p.write_text(ASCII.replace("3 0 3 1", "4 0 3 1 2"))
    with pytest.raises(ValueError, match="triangles"):
        mesh.read_ply(p)
    v = np.zeros(2, np.dtype([("x", "<f4"), ("y", "<f4"), ("z", "<f4")]))
    quad = np.array([(4, [0, 1, 1, 0])], np.dtype([("n", "u1"), ("v", "<i4", (4,))]))
    p.write_bytes(b"ply\nformat binary_little_endian 1.0\nelement vertex 2\nproperty float x\nproperty float y\n"
                  b"property float z\nelement face 1\nproperty list uchar int vertex_indices\nend_header\n"
                  + v.tobytes() + quad.tobytes())
    with pytest.raises(ValueError, match="triangle"):
        mesh.read_ply(p)
    p.write_bytes(b"ply\nformat binary_little_endian 1.0\nelement vertex 2\nproperty float x\nproperty float y\n"
                  b"property float z\nproperty list uchar int ids\nend_header\n" + bytes(40))
    with pytest.raises(ValueError, match="list"):
        mesh.read_ply(p)


# ------------------------------------------------------------------------------------------------ metrics
def test_metric_formulas():
    from sparf_b200 import mesh
    inf = float("inf")
    acc = torch.tensor([0.0, 0.1, 0.2, 0.4])
    comp = torch.tensor([0.05, 0.3, inf])
    m = mesh.distance_metrics(acc, comp, 0.25)
    assert m["accuracy"] == pytest.approx(0.175) and m["completeness"] == inf and m["chamfer"] == inf
    assert m["precision"] == 0.75 and m["recall"] == pytest.approx(1 / 3)
    assert m["fscore"] == pytest.approx(2 * 0.75 / 3 / (0.75 + 1 / 3)) and m["hausdorff"] == inf
    assert (m["n_pred"], m["n_ref"]) == (4, 3)
    m = mesh.distance_metrics(acc, comp, 0.25, max_dist=0.5)
    assert m["completeness"] == pytest.approx((0.05 + 0.3 + 0.5) / 3) and m["hausdorff"] == 0.5
    assert m["chamfer"] == pytest.approx((0.175 + 0.85 / 3) / 2)
    m = mesh.distance_metrics(acc, comp, 0.01)       # only the exact zero is below
    assert m["precision"] == 0.25 and m["recall"] == 0.0 and m["fscore"] == pytest.approx(0.0)
    m = mesh.distance_metrics(acc, comp, 0.0)
    assert m["fscore"] == 0.0
    m = mesh.distance_metrics(torch.zeros(0), torch.full((5,), inf), 0.1, max_dist=2.0)
    assert math.isnan(m["accuracy"]) and m["completeness"] == 2.0 and m["precision"] == 0 and m["recall"] == 0
    assert m["fscore"] == 0 and m["hausdorff"] == 2.0 and m["n_pred"] == 0


# ------------------------------------------------------------------------------------------------ argument checks
def _no_library_call(monkeypatch):
    from sparf_b200 import _lib

    def refuse():
        raise AssertionError("the library was called")
    monkeypatch.setattr(_lib, "lib", refuse)


def test_distance_grid_rejects_bad_arguments(monkeypatch):
    from sparf_b200 import ops
    _no_library_call(monkeypatch)
    v = torch.zeros(5, 3, device="meta")
    f = torch.zeros(4, 3, dtype=torch.int64, device="meta")
    bad = [dict(vertices=v.double()), dict(vertices=v[:, :2]), dict(vertices=v[0]), dict(vertices=None),
           dict(faces=f.int()), dict(faces=f[:, :2]), dict(vertices=v[:0]), dict(cells=0), dict(cells=(2, 2)),
           dict(cells=(1, 1, -1)), dict(cells=True), dict(cells=1.5), dict(cells=257), dict(cells=(4096, 4096, 2)),
           dict(vertices=torch.zeros(5, 3)), dict(faces=torch.zeros(4, 3, dtype=torch.int64))]
    for b in bad:
        kw = dict(dict(vertices=v, faces=f, cells=None), **b)
        with pytest.raises(ValueError):
            ops.distance_grid(kw["vertices"], kw["faces"], cells_per_axis=kw["cells"])
    with pytest.raises(ValueError, match="CUDA"):
        ops.distance_grid(torch.zeros(5, 3))
    with pytest.raises(ValueError, match="CUDA"):
        ops.distance_grid(torch.zeros(5, 3), torch.zeros(4, 3, dtype=torch.int64))


def test_closest_points_rejects_bad_arguments(monkeypatch):
    from sparf_b200 import ops
    _no_library_call(monkeypatch)
    v = torch.zeros(5, 3, device="meta")
    g = ops.DistanceGrid(v, None, None, None, None, (1, 1, 1), 0)
    p = torch.zeros(7, 3, device="meta")
    for args in [(None, p), (g, p.double()), (g, p[:, :2]), (g, p[0]), (g, torch.zeros(7, 3)), (g, p, -1.0),
                 (g, p, float("nan")), (g, p, "1")]:
        with pytest.raises(ValueError):
            ops.closest_points(*args)


def test_compare_and_sampling_reject_bad_arguments(monkeypatch):
    from sparf_b200 import mesh
    _no_library_call(monkeypatch)
    m = dict(vertices=torch.zeros(3, 3), faces=torch.tensor([[0, 1, 2]]))
    for kw in (dict(threshold=0.0), dict(threshold=-1.0), dict(threshold=1.0, max_dist=-1.0),
               dict(threshold=float("nan"))):
        with pytest.raises(ValueError):
            mesh.compare(m, m, **kw)
    for n in (-1, 1.5, True):
        with pytest.raises(ValueError):
            mesh.sample_surface(m, n)


def test_sample_surface_on_the_cpu():
    """area weighting and barycentrics (the function is plain torch: it runs on any device)"""
    from sparf_b200 import mesh
    v = torch.tensor([[0, 0, 0], [1, 0, 0], [0, 1, 0], [10, 0, 0], [13, 0, 0], [10, 3, 0], [5, 5, 5]], dtype=torch.float32)
    f = torch.tensor([[0, 1, 2], [3, 4, 5], [6, 6, 6]])
    p = mesh.sample_surface(dict(vertices=v, faces=f), 20000, seed=3)
    assert p.shape == (20000, 3) and p.dtype == torch.float32 and (p[:, 2] == 0).all()
    big = p[:, 0] >= 10
    assert abs(big.float().mean().item() - 0.9) < 0.01          # areas 0.5 and 4.5
    q = p[big] - torch.tensor([10.0, 0, 0])
    assert (q >= 0).all() and (q[:, 0] + q[:, 1] <= 3 + 1e-5).all()
    assert abs(q[:, 0].mean().item() - 1.0) < 0.03                # the centroid
    assert torch.equal(p, mesh.sample_surface(dict(vertices=v, faces=f), 20000, seed=3))
    assert mesh.sample_surface(dict(vertices=v, faces=f[2:]), 10).shape == (0, 3)
    assert mesh.sample_surface(dict(vertices=v, faces=f[:0]), 10).shape == (0, 3)


# ------------------------------------------------------------------------------------------------ declaration, binding
def test_declared_and_bound():
    from sparf_b200 import _lib
    src = open(os.path.join(ROOT, "include", "sparf_b200.h")).read()
    for name in ENTRY_POINTS:
        assert name + "(" in src, name
        assert name in _lib.exported_symbols(), name
    L = _lib.lib()
    for name in ENTRY_POINTS:
        assert hasattr(L, name), name


def test_c_entry_points_reject_invalid_sizes():
    """SPARF_ERR_INVALID before anything is read or launched (the pointers are host dummies)"""
    from sparf_b200 import _lib
    L = _lib.lib()
    buf = (ctypes.c_int64 * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    for V, F in ((-1, 0), (1 << 31, 0), (5, -2), (5, 1 << 31), (0, 1)):
        assert L.sparf_distance_grid_count(p, V, p, F, 0, 0, 0, p, p, p, 1 << 20, None) == INVALID, (V, F)
        assert L.sparf_last_error()
        assert L.sparf_distance_grid_fill(p, V, p, F, p, 1, 0, p, p, p, 1 << 20, None) == INVALID, (V, F)
        assert L.sparf_distance_query(p, V, p, F, p, p, p, p, 1, 1.0, p, p, p, None) == INVALID, (V, F)
    for n, e in ((-1, 0), (1 << 31, 0), (5, -1), (5, 1 << 31)):
        assert L.sparf_distance_grid_workspace_bytes(n, e) == 0, (n, e)
    for cells in ((0, 0, 1), (-1, 1, 1), (4096, 4096, 2)):
        assert L.sparf_distance_grid_count(p, 5, p, 3, *cells, p, p, p, 1 << 20, None) == INVALID, cells
    assert L.sparf_distance_grid_count(p, 5, None, 3, 0, 0, 0, p, p, p, 1 << 20, None) == INVALID
    assert L.sparf_distance_grid_count(p, 5, p, 3, 0, 0, 0, None, p, p, 1 << 20, None) == INVALID
    assert L.sparf_distance_grid_count(None, 5, None, -1, 0, 0, 0, p, p, p, 1 << 20, None) == INVALID
    assert L.sparf_distance_grid_fill(p, 5, p, 3, p, 0, 4, p, p, p, 1 << 20, None) == INVALID        # no cells
    assert L.sparf_distance_grid_fill(p, 5, p, 3, p, (1 << 24) + 1, 4, p, p, p, 1 << 20, None) == INVALID
    assert L.sparf_distance_grid_fill(p, 5, p, 3, p, 8, 1 << 31, p, p, p, 1 << 20, None) == INVALID
    assert L.sparf_distance_grid_fill(p, 5, p, 3, None, 8, 4, p, p, p, 1 << 20, None) == INVALID
    assert L.sparf_distance_grid_fill(p, 5, p, 3, p, 8, 4, p, None, p, 1 << 20, None) == INVALID
    for md in (-1.0, float("nan")):
        assert L.sparf_distance_query(p, 5, p, 3, p, p, p, p, 1, md, p, p, p, None) == INVALID, md
    assert L.sparf_distance_query(p, 5, p, 3, p, p, p, p, -1, 1.0, p, p, p, None) == INVALID
    assert L.sparf_distance_query(p, 5, p, 3, p, p, p, None, 1, 1.0, p, p, p, None) == INVALID
    assert L.sparf_distance_query(p, 5, p, 3, None, p, p, p, 1, 1.0, p, p, p, None) == INVALID
    assert L.sparf_distance_query(p, 5, None, 3, p, p, p, p, 1, 1.0, p, p, p, None) == INVALID


# ------------------------------------------------------------------------------------------------ the tool
def test_tool_arguments_parse():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import compare_mesh as tool
    ap = tool.build_parser()
    a = tool.parse_args(ap, ["p.ply", "r.ply", "--threshold", "0.01"])
    assert (a.pred, a.ref, a.threshold, a.samples, a.max_dist, a.seed) == ("p.ply", "r.ply", 0.01, 1_000_000,
                                                                            float("inf"), 0)
    a = tool.parse_args(ap, ["p.ply", "r.ply", "--threshold", "2", "--samples", "10", "--max-dist", "5", "--seed", "3"])
    assert (a.samples, a.max_dist, a.seed) == (10, 5.0, 3)
    for bad in ([], ["p.ply", "r.ply"], ["p.ply", "r.ply", "--threshold", "0"], ["p.ply", "r.ply", "--threshold", "1",
                "--samples", "-1"], ["p.ply", "r.ply", "--threshold", "1", "--max-dist", "-2"]):
        with pytest.raises(SystemExit):
            tool.parse_args(ap, bad)
