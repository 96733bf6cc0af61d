"""Marching cubes without a GPU: the library's case table (sparf_mcubes_table) and the NumPy oracle built on it
(tests/mcubes_oracle.py) give closed, consistently oriented meshes; the density lattice and world mapping of
sparf_b200.mesh are BARF's; write_ply round-trips; sparf_mcubes_workspace_bytes is sane for large extents."""
import numpy as np
import pytest
import torch

import mcubes_oracle as O


@pytest.fixture(scope="module")
def table():
    return O.case_table()


def _random_pm1(rng, shape, border_outside):
    v = np.where(rng.random(shape) < 0.5, 1.0, -1.0).astype(np.float32)
    if border_outside:
        v[[0, -1]] = -1
        v[:, [0, -1]] = -1
        v[:, :, [0, -1]] = -1
    return v


def test_table_sanity(table):
    assert table.shape == (256, 15)
    assert (table[0] == -1).all() and (table[255] == -1).all()
    for c in range(256):
        row = table[c]
        n = int((row >= 0).sum())
        assert n % 3 == 0 and (row[:n] >= 0).all() and (row[n:] == -1).all(), c      # -1 only as padding
        used, crossing = set(row[:n].tolist()), set(O.crossing_edges(c))
        assert used == crossing, (c, sorted(used), sorted(crossing))
        tris = row[:n].reshape(-1, 3)
        assert all(len(set(t)) == 3 for t in tris.tolist()), c


def test_closed_and_oriented_on_random_volumes_with_every_case(table):
    """random +-1 volumes (iso 0) whose border is outside: every one of the 256 cases occurs, and the mesh is closed and
    consistently oriented every time"""
    seen = set()
    for seed in range(24):
        rng = np.random.default_rng(seed)
        vol = _random_pm1(rng, (12, 11, 13), border_outside=True)
        seen |= set(np.unique(O.cell_cases(vol, 0.0)).tolist())
        verts, faces = O.marching_cubes(vol, 0.0, table)
        assert len(faces) and O.is_closed_and_oriented(faces), seed
        assert faces.max() < len(verts) and len(np.unique(faces)) == len(verts)
    assert seen == set(range(256)), sorted(set(range(256)) - seen)


def test_open_volumes_and_single_cells_run(table):
    """inside points on the border (an open mesh) and the 256 single-cell volumes: valid ids, every vertex referenced"""
    vols = [_random_pm1(np.random.default_rng(100 + s), (7, 9, 5), border_outside=False) for s in range(8)]
    for c in range(256):
        vols.append(np.array([1.0 if c >> q & 1 else -1.0 for q in range(8)], np.float32).reshape(2, 2, 2).transpose(2, 1, 0))
    for i, vol in enumerate(vols):
        verts, faces = O.marching_cubes(vol, 0.0, table)
        assert verts.dtype == np.float32 and faces.dtype == np.int64
        if i >= 8:
            c = i - 8
            assert O.cell_cases(vol, 0.0).item() == c
            assert len(faces) == (table[c] >= 0).sum() // 3 and len(verts) == len(O.crossing_edges(c))
        if len(faces):
            assert faces.min() >= 0 and len(np.unique(faces)) == len(verts)


def test_density_lattice_is_barfs():
    """the slabs of density_grid are BARF's lattice stack(meshgrid(linspace(r0, r1, res + 1))), axis 0 = x, bit for bit"""
    from sparf_b200 import mesh
    for res, rng, rows in ((16, (-1.2, 1.2), 3), (37, (-0.7, 2.1), 5), (20, (-1.2, 1.2), 100)):
        t = mesh.lattice_axis(res, rng)
        assert t.dtype == torch.float32 and torch.equal(t, torch.linspace(rng[0], rng[1], res + 1))
        barf = torch.stack(torch.meshgrid(t, t, t, indexing="ij"), dim=-1)
        slabs = list(mesh.lattice_slabs(t, rows))
        assert [i0 for i0, _ in slabs] == list(range(0, res + 1, rows))
        got = torch.cat([p for _, p in slabs]).view(res + 1, res + 1, res + 1, 3)
        assert torch.equal(got, barf)
        assert torch.equal(got[3, 1, 2], torch.stack([t[3], t[1], t[2]]))


def test_trimesh_settings_and_world_mapping():
    from sparf_b200 import mesh
    from sparf_b200.utils.edict import edict
    assert mesh.trimesh_settings(edict()) == (128, (-1.2, 1.2), 25.0)
    opt = edict(trimesh=edict(res=64, range=[-2.0, 1.5], thres=3.5, chunk_size=16384))
    assert mesh.trimesh_settings(opt) == (64, (-2.0, 1.5), 3.5)
    assert mesh.trimesh_settings(opt, res=32, range=(0, 1)) == (32, (0.0, 1.0), 3.5)
    v = torch.rand(1000, 3) * 64
    assert torch.equal(mesh.to_world(v, 64, (-2.0, 1.5)), v / 64 * (1.5 - -2.0) + -2.0)
    # lattice point i maps onto the lattice coordinate t[i] (up to the rounding of two different fp32 formulas)
    t = mesh.lattice_axis(64, (-2.0, 1.5))
    idx = torch.arange(65, dtype=torch.float32)
    assert (mesh.to_world(idx, 64, (-2.0, 1.5)) - t).abs().max().item() < 1e-6


@pytest.mark.parametrize("normals", [False, True])
def test_write_ply_round_trip(tmp_path, normals):
    from sparf_b200 import mesh
    g = torch.Generator().manual_seed(3)
    v = torch.randn(57, 3, generator=g)
    f = torch.randint(0, 57, (91, 3), generator=g)
    n = torch.nn.functional.normalize(torch.randn(57, 3, generator=g), dim=-1) if normals else None
    path = str(tmp_path / "m.ply")
    mesh.write_ply(path, v, f, n)
    props, faces = O.read_ply(path)
    assert list(props) == ["x", "y", "z"] + (["nx", "ny", "nz"] if normals else [])
    assert np.array_equal(np.stack([props[k] for k in "xyz"], 1), v.numpy())
    if normals:
        assert np.array_equal(np.stack([props[k] for k in ("nx", "ny", "nz")], 1), n.numpy())
    assert np.array_equal(faces, f.numpy())
    mesh.write_ply(path, np.zeros((0, 3)), np.zeros((0, 3), np.int64))      # an empty mesh is a valid file
    props, faces = O.read_ply(path)
    assert len(props["x"]) == 0 and faces.shape == (0, 3)


def test_workspace_bytes_monotone_and_64_bit():
    """8 B per lattice point + 16 B per 2048 points (up to alignment), monotone, no overflow past 2^32 points; 0 for an
    extent below 2.  Nothing is allocated."""
    from sparf_b200 import _lib
    L = _lib.lib()
    for bad in ((1, 5, 5), (5, 1, 5), (5, 5, 0), (-3, 4, 4)):
        assert L.sparf_mcubes_workspace_bytes(*bad) == 0
    prev = 0
    for n in [2, 3, 64, 129, 513, 1024, 1625, 1626, 1999, 2000, 2001, 2048, 2049]:
        b = L.sparf_mcubes_workspace_bytes(n, n, n)
        pts = n ** 3
        assert b >= 8 * pts + 16 * (-(-pts // 2048)) and b <= 8 * pts + 16 * (-(-pts // 2048)) + 512, (n, b)
        assert b >= prev
        prev = b
    assert L.sparf_mcubes_workspace_bytes(2000, 2000, 2001) > L.sparf_mcubes_workspace_bytes(2000, 2000, 2000)
    assert L.sparf_mcubes_workspace_bytes(1 << 20, 1 << 20, 1 << 20) == 0      # 2^60 points: refused, not wrapped
