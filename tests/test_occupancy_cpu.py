"""Occupancy grids without a GPU: properties of the NumPy restatement (tests/occupancy_oracle.py) that the GPU tests hold
the kernels to, the C ABI's new entry points and workspace sizes, and OccupancyGrid's bookkeeping."""
import itertools

import numpy as np
import pytest
import torch

import occupancy_oracle as O


def _window_occupied(sigma, thres):
    """the rule spelled out per cell: any lattice point with indices in [c-1, c+2] per axis, clipped, >= thres or NaN"""
    res = sigma.shape[0] - 1
    out = np.zeros((res,) * 3, bool)
    for i, j, k in itertools.product(range(res), repeat=3):
        w = sigma[max(i - 1, 0):i + 3, max(j - 1, 0):j + 3, max(k - 1, 0):k + 3]
        out[i, j, k] = bool(((w >= thres) | np.isnan(w)).any())
    return out


@pytest.mark.parametrize("res,p", [(1, (0, 0, 1)), (2, (1, 2, 0)), (6, (3, 3, 3)), (6, (0, 6, 2)), (9, (9, 0, 4))])
def test_single_point_marks_the_cells_within_one_cell(res, p):
    thres = np.float32(0.25)
    sigma = np.zeros((res + 1,) * 3, np.float32)
    sigma[p] = thres
    occ = O.occupied_cells(sigma, thres)
    # cells touching p are p-1 and p per axis; with their neighbours: p-2 ... p+1, clipped to the grid
    want = np.zeros_like(occ)
    want[tuple(slice(max(q - 2, 0), min(q + 2, res)) for q in p)] = True
    assert np.array_equal(occ, want)
    assert np.array_equal(O.unpack_bits(O.build(sigma, thres), res), want)


def test_threshold_equality_and_nan_count_as_occupied():
    res = 6
    thres = np.float32(0.5)
    for v, occupied in ((thres, True), (np.nextafter(thres, np.float32(0)), False), (np.float32(np.nan), True),
                        (np.float32(np.inf), True), (np.float32(-np.inf), False)):
        sigma = np.zeros((res + 1,) * 3, np.float32)
        sigma[3, 3, 3] = v
        assert O.occupied_cells(sigma, thres).any() == occupied, v


def test_dilation_matches_the_per_cell_rule():
    rng = np.random.default_rng(3)
    for res in (1, 2, 5, 8):
        sigma = rng.random((res + 1,) * 3).astype(np.float32)
        sigma[rng.random(sigma.shape) < 0.03] = np.nan
        assert np.array_equal(O.occupied_cells(sigma, 0.97), _window_occupied(sigma, np.float32(0.97)))


def test_bit_packing_layout():
    res = 5
    occ = np.zeros((res,) * 3, bool)
    occ[1, 2, 3] = True                      # idx = (1*5 + 2)*5 + 3 = 38: word 1, bit 6
    bits = O.pack_bits(occ)
    assert bits.dtype == np.uint32 and bits.shape == (4,)
    assert bits.tolist() == [0, 1 << 6, 0, 0]
    assert np.array_equal(O.unpack_bits(bits, res), occ)


def test_box_faces():
    """u = res (x = r1) is outside and always kept; x = r0 is inside, in cell 0; just inside r1 is in the last cell; below
    r0 and NaN are kept"""
    res, r0, r1 = 4, -1.0, 1.0
    empty = O.pack_bits(np.zeros((res,) * 3, bool))
    o = np.array([[0.0, 0.0, 0.0], [r1, 0.0, 0.0], [r0, r0, r0], [0.0, 0.99, 0.0],
                  [np.nextafter(np.float32(r0), np.float32(-2)), 0.0, 0.0], [0.0, 0.0, np.nan]], np.float32)
    d = np.zeros_like(o)
    t = np.zeros((len(o), 1), np.float32)
    assert O.kept(empty, res, r0, r1, o, d, t)[:, 0].tolist() == [False, True, False, False, True, True]
    occ = np.zeros((res,) * 3, bool)
    occ[0, 0, 0] = True
    assert O.kept(O.pack_bits(occ), res, r0, r1, o, d, t)[:, 0].tolist() == [False, True, True, False, True, True]


def test_lookup_uses_the_encoder_op_order():
    """x = o + (d * t) with each op rounded to fp32, then (x - r0) / (r1 - r0) * res"""
    rng = np.random.default_rng(5)
    res, r0, r1 = 7, -0.7, 1.9
    o = rng.uniform(-1, 2, (50, 3)).astype(np.float32)
    d = rng.normal(size=(50, 3)).astype(np.float32)
    t = rng.uniform(0, 1, (50, 9)).astype(np.float32)
    occ = rng.random((res,) * 3) < 0.4
    keep = O.kept(O.pack_bits(occ), res, r0, r1, o, d, t)
    for r, k in itertools.product(range(50), range(9)):
        x = [np.float32(o[r, a] + np.float32(d[r, a] * t[r, k])) for a in range(3)]
        u = [np.float32(np.float32(x[a] - np.float32(r0)) / np.float32(np.float32(r1) - np.float32(r0))) * np.float32(res)
             for a in range(3)]
        inside = all(0 <= q < res for q in u)
        assert keep[r, k] == (not inside or occ[int(u[0]), int(u[1]), int(u[2])])
    idx, ok, dk, tk = O.compact(O.pack_bits(occ), res, r0, r1, o, d, t)
    assert np.array_equal(idx, np.flatnonzero(keep)) and np.array_equal(tk[:, 0], t.reshape(-1)[idx])
    assert np.array_equal(ok, o[idx // 9]) and np.array_equal(dk, d[idx // 9])


def test_abi_declares_the_occupancy_entry_points():
    import test_abi
    from sparf_b200 import _lib
    names = {"sparf_occupancy_build", "sparf_occupancy_workspace_bytes", "sparf_occupancy_count", "sparf_occupancy_emit"}
    assert names <= set(test_abi._header_functions())
    assert names <= set(_lib.exported_symbols())


def test_workspace_bytes():
    from sparf_b200 import _lib
    L = _lib.lib()
    for R, S in ((1, 1), (3, 700), (1000, 37), (524293, 4096), (1 << 40, 64)):
        tiles = -(-R * S // 2048)
        assert L.sparf_occupancy_workspace_bytes(R, S) == -(-tiles * 2048 // 256) * 256 + 8 * tiles, (R, S)
    assert L.sparf_occupancy_workspace_bytes(-1, 4) == 0 and L.sparf_occupancy_workspace_bytes(4, 0) == 0
    assert L.sparf_occupancy_workspace_bytes(1 << 40, 1 << 20) == 0          # above 2^58 samples


def test_occupied_fraction():
    from sparf_b200.occupancy import OccupancyGrid
    rng = np.random.default_rng(9)
    for res in (1, 3, 8):
        occ = rng.random((res,) * 3) < 0.3
        g = OccupancyGrid(torch.from_numpy(O.pack_bits(occ).view(np.int32).copy()), res, (-1.2, 1.2), 0.01)
        assert g.occupied_fraction() == occ.mean()
