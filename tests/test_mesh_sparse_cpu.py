"""Sparse marching cubes without a GPU: the NumPy restatement (tests/sparse_mcubes_oracle.py) classifies blocks by
the rule of include/sparf_b200.h, its block-wise mesh equals the dense oracle restricted to the active blocks (and the
dense oracle itself with every block active), res must be a multiple of 8, and the workspace query refuses invalid
sizes."""
import numpy as np
import pytest

import mcubes_oracle as O
import sparse_mcubes_oracle as S


@pytest.fixture(scope="module")
def table():
    return O.case_table()


def _sphere(res, radius, center):
    x = np.stack(np.meshgrid(*[np.arange(res + 1, dtype=np.float64)] * 3, indexing="ij"), -1)
    return (radius - np.linalg.norm(x - center, axis=-1)).astype(np.float32)


def _equal(a, b):
    (av, af), (bv, bf) = a, b
    assert av.shape == bv.shape and af.shape == bf.shape, (av.shape, bv.shape, af.shape, bf.shape)
    assert np.array_equal(av.view(np.uint32), bv.view(np.uint32)) and np.array_equal(af, bf)


def test_classification_rule():
    rng = np.random.default_rng(0)
    nb = 5
    coarse = rng.standard_normal((nb + 1,) * 3).astype(np.float32)
    coarse[2, 3, 1] = np.nan
    act = S.classify(coarse, 0.4)
    for b in np.ndindex(nb, nb, nb):
        w = coarse[tuple(slice(max(x - 1, 0), min(x + 2, nb) + 1) for x in b)]
        expect = np.isnan(w).any() or ((w >= 0.4).any() and (w < 0.4).any())
        assert act[b] == expect, b
    assert act[1:4, 2:5, 0:3].all()                                  # every window around the NaN
    assert not S.classify(np.full((4, 4, 4), 2.0, np.float32), 1.0).any()
    assert not S.classify(np.full((4, 4, 4), 0.0, np.float32), 1.0).any()


def test_block_mesh_equals_filtered_dense_on_random_pm1(table):
    """random ±1 volumes (all 256 cases) under random active subsets, and all blocks active = the dense oracle"""
    seen = set()
    res, nb = 24, 3
    for seed in range(6):
        rng = np.random.default_rng(seed)
        vol = np.where(rng.random((res + 1,) * 3) < 0.5, 1.0, -1.0).astype(np.float32)
        seen |= set(np.unique(O.cell_cases(vol, 0.0)).tolist())
        for frac in (0.3, 0.7, 1.0):
            active = rng.random((nb,) * 3) < frac if frac < 1 else np.ones((nb,) * 3, bool)
            ids = np.flatnonzero(active.reshape(-1))
            got = S.marching_cubes_blocks(S.block_points(vol, ids, nb), ids, res, 0.0, table)
            _equal(got, S.dense_filtered(vol, 0.0, active, table))
            if frac == 1.0:
                _equal(got, O.marching_cubes(vol, 0.0, table))
    assert seen == set(range(256))


def test_sphere_all_crossings_active_equals_dense(table):
    """a smooth surface: the classified blocks hold every crossing cell, so the sparse mesh is the dense one; an empty
    block set gives an empty mesh"""
    res = 48
    vol = _sphere(res, 14.3, np.array([23.2, 24.7, 22.9]))
    active = S.classify(vol[::8, ::8, ::8], 0.0)
    assert 0 < active.sum() < active.size
    ids = np.flatnonzero(active.reshape(-1))
    got = S.marching_cubes_blocks(S.block_points(vol, ids, res // 8), ids, res, 0.0, table)
    _equal(got, O.marching_cubes(vol, 0.0, table))
    assert O.is_closed_and_oriented(got[1]) and O.euler_characteristic(got[1]) == 2
    v, f = S.marching_cubes_blocks(np.zeros((0, 9, 9, 9), np.float32), [], res, 0.0, table)
    assert v.shape == (0, 3) and f.shape == (0, 3)


def test_res_must_be_a_multiple_of_8():
    from sparf_b200 import mesh
    from sparf_b200.utils.edict import edict
    for res in (0, 4, 12, 100, 129):
        with pytest.raises(ValueError):
            mesh.check_sparse_res(res)
        with pytest.raises(ValueError):
            mesh.extract_mesh_sparse(edict(trimesh=edict(res=res, range=[-1.2, 1.2], thres=1.0)), None)
    for res in (8, 128, 2048):
        mesh.check_sparse_res(res)


def test_workspace_refuses_invalid_sizes():
    """0 for a res that is no multiple of 8 or beyond 8192, more active blocks than blocks, negative sizes, and lengths
    past cub's 32-bit item counts (no wrap-around)"""
    from sparf_b200 import _lib
    L = _lib.lib()
    for res, n, v in ((0, 0, 0), (7, 0, 0), (12, 0, 0), (8200, 0, 0), (-8, 0, 0), (16, 9, 0), (16, -1, 0), (16, 1, -1),
                      (16, 1, 1 << 31), (8192, 1 << 25, 0), (8192, 1 << 40, 0), (1 << 30, 0, 0)):
        assert L.sparf_mcubes_sparse_workspace_bytes(res, n, v) == 0, (res, n, v)


def test_emit_refuses_a_face_capacity_past_the_bound():
    """emit's face capacity is at most 5 triangles per cell of the active blocks (2560 per block): a larger one is the
    caller's error and is refused before any device work"""
    from sparf_b200 import _lib
    L = _lib.lib()
    for n, cap in ((1, 2561), (3, 3 * 2560 + 1), (1, 1 << 40), (0, 1), (1, -1)):
        rc = L.sparf_mcubes_sparse_emit(None, 16, None, None, n, 0.0, 0, cap, None, None, None, 0, None)
        assert rc == 1, (n, cap, rc)
