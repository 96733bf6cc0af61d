"""CPU checks of the mesh simplification: the oracle on hand-worked meshes, argument checks that fail before any
library call, the C entries' refusals, the declarations and bindings, and the tool's flag."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

import simplify_oracle as SO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INVALID = 1     # SPARF_ERR_INVALID
ENTRY_POINTS = ["sparf_mesh_simplify_workspace_bytes", "sparf_mesh_simplify_init", "sparf_mesh_simplify_round",
                "sparf_mesh_simplify_emit"]

OCTAHEDRON = (np.array([[1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1]], np.float32),
              np.array([[0, 2, 4], [2, 1, 4], [1, 3, 4], [3, 0, 4], [2, 0, 5], [1, 2, 5], [3, 1, 5], [0, 3, 5]]))
TETRAHEDRON = (np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]], np.float32),
               np.array([[0, 2, 1], [0, 1, 3], [0, 3, 2], [1, 2, 3]]))


# ------------------------------------------------------------------------------------------------ the oracle
def test_octahedron_collapses_to_a_tetrahedron():
    """8 faces: 2 collapses leave 4 faces, and the tetrahedron that remains takes no collapse"""
    v, f = OCTAHEDRON
    vo, fo, ids, _, rounds = SO.simplify(v, f, 0)
    assert fo.shape == (4, 3) and len(ids) == 4 and len(vo) == 4
    assert (len(vo) - 6 + len(fo)) == 2      # Euler: V - E + F with E = 6
    vo, fo, ids, _, _ = SO.simplify(v, f, 6)
    assert fo.shape == (6, 3) and len(ids) == 5


def test_tetrahedron_is_kept_by_the_link_condition():
    v, f = TETRAHEDRON
    vo, fo, ids, _, rounds = SO.simplify(v, f, 0)
    assert np.array_equal(fo, f) and np.array_equal(ids, np.arange(4)) and vo.tobytes() == v.tobytes()
    assert rounds == 1          # one round finds no valid edge


def test_two_triangle_square_is_unchanged():
    """all four vertices are on the boundary, so no edge may collapse"""
    v = np.array([[0, 0, 0], [1, 0, 0], [1, 1, 0], [0, 1, 0]], np.float32)
    f = np.array([[0, 1, 2], [0, 2, 3]])
    vo, fo, ids, _, rounds = SO.simplify(v, f, 0)
    assert np.array_equal(fo, f) and vo.tobytes() == v.tobytes() and rounds == 1


def test_fold_check_rejects_the_cheapest_edge():
    """a flat fan: every cost is 0, so the cheapest key is edge 0, (hub, 1).  Moving the hub onto vertex 1 would turn
    the face (hub, 5, 6) over (vertex 1 lies beyond the line 5-6), so that edge is not valid"""
    v = np.array([[0, 0, 0], [1, 0, 0], [.5, .866, 0], [-.5, .866, 0], [-1, 0, 0], [0, -1, 0], [.3, -.1, 0]],
                 np.float32)
    f = np.array([[0, k, k % 6 + 1] for k in range(1, 7)])
    pos, Q, fl = SO.setup(v, f)
    edges, _, _, bnd, keys = SO.classify(pos, Q, fl)
    assert edges[0] == (0, 1) and bnd[1] and not bnd[0]
    valid = [edges[k & 0xffffffff] for k in keys]
    assert (0, 1) not in valid and (0, 2) in valid
    assert all(k >> 32 == 0 for k in keys)
    vo, fo, ids, _, _ = SO.simplify(v, f, 0)
    assert ids.tolist() == [1, 2, 3, 4, 5, 6] and vo.tobytes() == v[1:].tobytes()     # the border kept exactly
    assert len(fo) == 4


def test_constant_attribute_is_exact():
    v, f = OCTAHEDRON
    a = np.full((6, 2), 0.3, np.float32)
    _, _, _, ao, _ = SO.simplify(v, f, 0, attrs=a)
    assert (ao == np.float32(0.3)).all()


# ------------------------------------------------------------------------------------------------ argument checks
def _no_library_call(monkeypatch):
    from sparf_b200 import _lib

    def refuse():
        raise AssertionError("the library was called")
    monkeypatch.setattr(_lib, "lib", refuse)


def test_mesh_simplify_rejects_bad_arguments(monkeypatch):
    from sparf_b200 import ops
    _no_library_call(monkeypatch)
    v = torch.zeros(5, 3, device="meta")
    f = torch.zeros(4, 3, dtype=torch.int64, device="meta")
    a = torch.zeros(5, 2, device="meta")
    bad = [dict(vertices=v.double()), dict(vertices=v[:, :2]), dict(vertices=v[0]), dict(vertices=None),
           dict(faces=f.int()), dict(faces=f[:, :2]), dict(vertices=v[:0]), dict(target=-1), dict(target=1.5),
           dict(target=True), dict(attrs=a.double()), dict(attrs=a[:4]), dict(attrs=a[0]),
           dict(attrs=torch.zeros(5, 2)), dict(vertices=torch.zeros(5, 3))]
    for b in bad:
        kw = dict(dict(vertices=v, faces=f, target=2, attrs=a), **b)
        with pytest.raises(ValueError):
            ops.mesh_simplify(kw["vertices"], kw["faces"], kw["target"], attrs=kw["attrs"])
    with pytest.raises(ValueError, match="CUDA"):           # well formed, but not on a GPU
        ops.mesh_simplify(torch.zeros(5, 3), torch.zeros(4, 3, dtype=torch.int64), 2)
    with pytest.raises(ValueError):
        ops.mesh_simplify(v, torch.zeros(ops.MAX_SIMPLIFY_FACES + 1, 3, dtype=torch.int64, device="meta"), 2)


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
    for V, F, A in ((-1, 0, 0), (1 << 31, 0, 0), (5, -1, 0), (5, (1 << 31) // 3 + 1, 0), (0, 1, 0), (5, 3, -1)):
        assert L.sparf_mesh_simplify_workspace_bytes(V, F, A) == 0, (V, F, A)
        assert L.sparf_mesh_simplify_init(p, p, p, V, F, A, p, p, 1 << 20, None) == INVALID, (V, F, A)
        assert L.sparf_last_error()
        assert L.sparf_mesh_simplify_round(V, F, A, 0, 1, p, p, 1 << 20, None) == INVALID, (V, F, A)
        assert L.sparf_mesh_simplify_emit(V, F, A, 0, p, p, p, p, p, 1 << 20, None) == INVALID, (V, F, A)
    assert L.sparf_mesh_simplify_init(None, p, p, 5, 3, 1, p, p, 1 << 20, None) == INVALID
    assert L.sparf_mesh_simplify_init(p, None, p, 5, 3, 1, p, p, 1 << 20, None) == INVALID
    assert L.sparf_mesh_simplify_init(p, p, None, 5, 3, 1, p, p, 1 << 20, None) == INVALID
    assert L.sparf_mesh_simplify_init(p, p, p, 5, 3, 1, None, p, 1 << 20, None) == INVALID
    assert L.sparf_mesh_simplify_round(5, 3, 0, 4, 1, p, p, 1 << 20, None) == INVALID       # n_live > F
    assert L.sparf_mesh_simplify_round(5, 3, 0, 3, 0, p, p, 1 << 20, None) == INVALID       # k = 0
    assert L.sparf_mesh_simplify_round(5, 3, 0, 3, 1, None, p, 1 << 20, None) == INVALID
    assert L.sparf_mesh_simplify_emit(5, 3, 0, 3, p, p, p, None, p, 1 << 20, None) == INVALID
    assert L.sparf_mesh_simplify_emit(5, 3, 0, 3, None, p, p, p, p, 1 << 20, None) == INVALID


# ------------------------------------------------------------------------------------------------ the tool
def test_tool_flag_parses():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import extract_mesh as tool
    ap = tool.build_parser()
    assert tool.parse_args(ap, ["m.pth", "--out", "x.ply"]).simplify is None
    a = tool.parse_args(ap, ["m.pth", "--out", "x.ply", "--sparse", "--keep-largest", "1", "--simplify", "200000"])
    assert (a.simplify, a.keep_largest, a.sparse) == (200000, 1, True)
    assert tool.parse_args(ap, ["m.pth", "--out", "x.ply", "--tsdf", "c.npz", "--simplify", "0"]).simplify == 0
    for bad in (["--simplify", "-1"], ["--simplify", "x"]):
        with pytest.raises(SystemExit):
            tool.parse_args(ap, ["m.pth", "--out", "x.ply"] + bad)
