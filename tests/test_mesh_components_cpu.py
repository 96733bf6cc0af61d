"""CPU checks of the mesh components: the oracle against a breadth-first search and hand-worked meshes, argument checks
that fail before any library call, the declarations and bindings, and the tool's flags."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

import components_oracle as CO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INVALID = 1     # SPARF_ERR_INVALID
ENTRY_POINTS = ["sparf_mesh_components_workspace_bytes", "sparf_mesh_components", "sparf_mesh_component_faces",
                "sparf_mesh_select_count", "sparf_mesh_select_emit"]


# ------------------------------------------------------------------------------------------------ the oracle
@pytest.mark.parametrize("seed", range(6))
def test_oracle_matches_bfs_on_random_meshes(seed):
    rng = np.random.default_rng(seed)
    V = int(rng.integers(1, 200))
    f = CO.random_soup(V, int(rng.integers(0, 300)), seed, n_groups=int(rng.integers(1, 40)))
    labels, counts = CO.components(f, V)
    assert np.array_equal(labels, CO.bfs_labels(f, V))
    assert counts.sum() == len(f) and len(counts) == labels.max() + 1
    # the labels do not depend on the face order, nor on the vertex order within a face
    perm = rng.permutation(len(f))
    rot = np.roll(f[perm], int(rng.integers(0, 3)), axis=1)
    assert np.array_equal(CO.components(rot, V)[0], labels)


def test_oracle_hand_worked():
    # vertex 2 unused; faces {0,1,3} and {3,4,4} (degenerate) share vertex 3; {5,6,7}; vertex 8 unused
    f = np.array([[3, 4, 4], [5, 6, 7], [1, 0, 3]])
    labels, counts = CO.components(f, 9)
    assert labels.tolist() == [0, 0, 1, 0, 0, 2, 2, 2, 3]
    assert counts.tolist() == [2, 0, 1, 0]
    # two triangles sharing only a vertex are one component
    labels, counts = CO.components(np.array([[0, 1, 2], [2, 3, 4]]), 5)
    assert labels.tolist() == [0] * 5 and counts.tolist() == [2]
    # F = 0: every vertex its own component; V = 0: nothing
    labels, counts = CO.components(np.zeros((0, 3), np.int64), 4)
    assert labels.tolist() == [0, 1, 2, 3] and counts.tolist() == [0, 0, 0, 0]
    labels, counts = CO.components(np.zeros((0, 3), np.int64), 0)
    assert labels.shape == counts.shape == (0,)


def test_oracle_selection_hand_worked():
    f = np.array([[3, 4, 4], [5, 6, 7], [1, 0, 3]])
    labels, counts = CO.components(f, 9)
    keep = CO.keep_mask(counts, min_faces=1)
    assert keep.tolist() == [1, 0, 1, 0]
    vert_ids, faces = CO.select(f, labels, keep)
    assert vert_ids.tolist() == [0, 1, 3, 4, 5, 6, 7]
    assert faces.tolist() == [[2, 3, 3], [4, 5, 6], [1, 0, 2]]
    assert CO.keep_mask(counts, largest=1).tolist() == [1, 0, 0, 0]
    assert CO.keep_mask(counts, largest=1, min_faces=0).tolist() == [1, 0, 0, 0]
    # ties go to the smaller label
    assert CO.keep_mask(np.array([1, 3, 3, 2]), largest=2).tolist() == [0, 1, 1, 0]
    assert CO.keep_mask(counts, min_faces=0).tolist() == [1, 1, 1, 1]
    vert_ids, faces = CO.select(f, labels, np.zeros(4, np.uint8))
    assert vert_ids.shape == (0,) and faces.shape == (0, 3)


# ------------------------------------------------------------------------------------------------ argument checks
def _no_library_call(monkeypatch):
    from sparf_b200 import _lib

    def refuse():
        raise AssertionError("the library was called")
    monkeypatch.setattr(_lib, "lib", refuse)


def test_mesh_components_rejects_bad_arguments(monkeypatch):
    from sparf_b200 import ops
    _no_library_call(monkeypatch)
    good = torch.zeros(4, 3, dtype=torch.int64)
    bad = [(good.int(), 5), (good.float(), 5), (torch.zeros(4, 4, dtype=torch.int64), 5), (torch.zeros(12, dtype=torch.int64), 5),
           (good.numpy(), 5), (good, -1), (good, 2 ** 31), (good, 5.0), (good, True), (good, 0),
           (good, 5),                                   # well formed, but on the CPU
           (torch.zeros(4, 3, dtype=torch.int64, device="meta"), 5)]
    for faces, n in bad:
        with pytest.raises(ValueError):
            ops.mesh_components(faces, n)


def test_mesh_select_rejects_bad_arguments(monkeypatch):
    from sparf_b200 import ops
    _no_library_call(monkeypatch)
    f = torch.zeros(4, 3, dtype=torch.int64, device="meta")
    lab = torch.zeros(5, dtype=torch.int32, device="meta")
    keep = torch.ones(2, dtype=torch.uint8, device="meta")
    bad = [dict(labels=lab.long()), dict(labels=lab[:4]), dict(labels=None), dict(keep=keep.int()), dict(keep=keep[None]),
           dict(keep=torch.ones(6, dtype=torch.uint8, device="meta")), dict(keep=keep[:0]), dict(n_verts=-1),
           dict(faces=f.int()), dict(labels=torch.zeros(5, dtype=torch.int32))]
    for b in bad:
        kw = dict(dict(faces=f, n_verts=5, labels=lab, keep=keep), **b)
        with pytest.raises(ValueError):
            ops.mesh_select(kw["faces"], kw["n_verts"], kw["labels"], kw["keep"])
    with pytest.raises(ValueError, match="CUDA"):           # well formed, but not on a GPU
        ops.mesh_select(f, 5, lab, keep)


def test_keep_components_rejects_bad_arguments(monkeypatch):
    from sparf_b200 import mesh
    _no_library_call(monkeypatch)
    m = dict(vertices=torch.zeros(3, 3), faces=torch.tensor([[0, 1, 2]]))
    for kw in (dict(largest=0), dict(largest=-2), dict(largest=1.5), dict(largest=True), dict(min_faces=-1),
               dict(min_faces=0.5)):
        with pytest.raises(ValueError):
            mesh.keep_components(m, **kw)
    with pytest.raises(ValueError, match="CUDA"):
        mesh.keep_components(m, largest=1)


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
    big = 1 << 31
    for V, F in ((-1, 0), (big, 0), (5, -1), (5, big), (0, 1)):
        assert L.sparf_mesh_components_workspace_bytes(V, F) == 0, (V, F)
        assert L.sparf_mesh_components(p, F, V, p, p, p, 1 << 20, None) == INVALID, (V, F)
        assert L.sparf_last_error()
        assert L.sparf_mesh_component_faces(p, F, V, p, 0, p, None) == INVALID, (V, F)
        assert L.sparf_mesh_select_count(p, F, V, p, p, 0, p, p, 1 << 20, None) == INVALID, (V, F)
        assert L.sparf_mesh_select_emit(p, F, V, p, p, 0, p, p, p, 1 << 20, None) == INVALID, (V, F)
    assert L.sparf_mesh_components(None, 3, 5, p, p, p, 1 << 20, None) == INVALID
    assert L.sparf_mesh_components(p, 3, 5, None, p, p, 1 << 20, None) == INVALID
    assert L.sparf_mesh_component_faces(p, 3, 5, p, 6, p, None) == INVALID           # C > V
    assert L.sparf_mesh_component_faces(p, 3, 5, p, -1, p, None) == INVALID
    assert L.sparf_mesh_select_count(p, 3, 5, p, p, 6, p, p, 1 << 20, None) == INVALID
    assert L.sparf_mesh_select_count(p, 3, 5, p, None, 2, p, p, 1 << 20, None) == INVALID
    assert L.sparf_mesh_select_emit(p, 3, 5, None, p, 2, p, p, p, 1 << 20, None) == INVALID


# ------------------------------------------------------------------------------------------------ the tool
def test_tool_flags_parse():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import extract_mesh as tool
    ap = tool.build_parser()
    a = tool.parse_args(ap, ["m.pth", "--out", "x.ply"])
    assert a.keep_largest is None and a.min_faces is None
    a = tool.parse_args(ap, ["m.pth", "--out", "x.ply", "--keep-largest", "3", "--min-faces", "50", "--sparse"])
    assert (a.keep_largest, a.min_faces, a.sparse) == (3, 50, True)
    a = tool.parse_args(ap, ["m.pth", "--out", "x.ply", "--tsdf", "c.npz", "--min-faces", "0"])
    assert (a.keep_largest, a.min_faces, a.tsdf) == (None, 0, "c.npz")
    for bad in (["--keep-largest", "0"], ["--keep-largest", "x"], ["--min-faces", "-1"]):
        with pytest.raises(SystemExit):
            tool.parse_args(ap, ["m.pth", "--out", "x.ply"] + bad)
