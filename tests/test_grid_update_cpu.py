"""CPU-side checks of the occupancy grid update (occupancy.update_): the new entry points are declared in the header and
bound in the ctypes table, update_ rejects every bad argument before any library call, and the NumPy oracle's sampled
cells and points are what the semantics say."""
import os
import re

import numpy as np
import pytest
import torch

import grid_update_oracle as G
import occupancy_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ("sparf_occupancy_sample_workspace_bytes", "sparf_occupancy_sample", "sparf_occupancy_ema")


def test_entry_points_declared_and_bound():
    from sparf_b200 import _lib
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "sparf_b200.h")).read(), flags=re.S)
    for name in NEW:
        assert re.search(r"\b%s\s*\(" % name, src), name
        assert name in _lib.exported_symbols(), name


def _grid(res=8, contraction=None, density=True):
    from sparf_b200.occupancy import CONTRACTED_RANGE, OccupancyGrid
    bits = torch.full(((res ** 3 + 31) // 32,), -1, dtype=torch.int32)
    dens = torch.zeros(res ** 3) if density else None
    return OccupancyGrid(bits, res, CONTRACTED_RANGE if contraction else (-1.0, 1.0), 0.01, contraction, dens)


@pytest.fixture
def no_library(monkeypatch):
    """every path into the native library or the network raises"""
    from sparf_b200 import _lib, ops

    def boom(*a, **k):
        raise AssertionError("library call before the arguments were checked")
    monkeypatch.setattr(_lib, "lib", boom)
    for name in ("occupancy_sample", "occupancy_ema_", "density_forward"):
        monkeypatch.setattr(ops, name, boom)


@pytest.mark.parametrize("case", ["no_density", "decay_0", "decay_above_1", "decay_nan", "negative_uniform",
                                  "negative_occupied", "u_cell_shape", "u_jit_shape", "contracted_res_7"])
def test_update_rejects_bad_arguments(case, no_library):
    from sparf_b200 import occupancy
    grid, kw = _grid(), dict(n_uniform=4, n_occupied=4)
    if case == "no_density":
        grid = _grid(density=False)
    elif case == "decay_0":
        kw["decay"] = 0.0
    elif case == "decay_above_1":
        kw["decay"] = 1.5
    elif case == "decay_nan":
        kw["decay"] = float("nan")
    elif case == "negative_uniform":
        kw["n_uniform"] = -1
    elif case == "negative_occupied":
        kw["n_occupied"] = -1
    elif case == "u_cell_shape":
        kw["draws"] = (torch.rand(7), torch.rand(8, 3))
    elif case == "u_jit_shape":
        kw["draws"] = (torch.rand(8), torch.rand(8, 2))
    elif case == "contracted_res_7":
        grid = _grid(res=7, contraction=((0.0, 0.0, 0.0), 1.0))
    before = (grid.bits.clone(), None if grid.density is None else grid.density.clone())
    with pytest.raises(ValueError):
        occupancy.update_(grid, None, **kw)
    assert torch.equal(grid.bits, before[0])


@pytest.mark.parametrize("contraction", [None, ((0.25, -0.5, 1.0), 1.5)])
@pytest.mark.parametrize("res", [8, 33])
def test_oracle_points_map_back_into_their_cells(res, contraction):
    """each point's cell (box: (x - r0) / (r1 - r0) * res; contracted: the exact fp64 contraction) is its drawn cell,
    or its neighbour across a face where fp32 rounding moved a point on that face (jitter 0 or 1 - 2^-24) over it"""
    import contraction_oracle as C
    rng = np.random.default_rng(res)
    n = 4096
    cells = np.nonzero(G.interior(res, contraction is not None))[0]
    cells = cells[rng.integers(0, cells.size, n)]
    u_jit = rng.random((n, 3), dtype=np.float32)
    u_jit[:64] = 0.0
    u_jit[64:128] = np.float32(1 - 2 ** -24)
    r0, r1 = -1.3, 0.7
    x = G.points(cells, res, r0, r1, contraction, u_jit).astype(np.float64)
    if contraction is None:
        u = (x - float(np.float32(r0))) / (float(np.float32(r1)) - float(np.float32(r0))) * res
    else:
        c, r = contraction
        v = C.contract64((x - np.asarray(c, np.float32).astype(np.float64)) / float(np.float32(r)))
        u = (v + 2) / 4 * res
    got = np.floor(u).astype(np.int64)
    want = np.stack([cells // (res * res), cells // res % res, cells % res], -1)
    off = np.abs(got - want)
    at_face = (u_jit < 1e-4) | (u_jit > 1 - 1e-4)
    assert off.max() <= 1 and not (off.astype(bool) & ~at_face).any()
    assert (off.sum(-1) == 0).mean() > 0.9


def test_oracle_sampling_rules():
    """u_cell = (arange(I) + 0.5) / I visits every interior cell once in increasing order; the occupied half draws only
    occupied interior cells; with none occupied it falls back to the uniform rule"""
    res = 9
    inner = np.nonzero(G.interior(res, True))[0]
    I = inner.size
    assert I == (res - 4) ** 3
    occ = np.random.default_rng(0).random((res,) * 3) < 0.3
    bits = O.pack_bits(occ)
    u = ((np.arange(I) + 0.5) / I).astype(np.float32)
    cells, _ = G.sample(bits, res, 0, 0, ((0.0, 0.0, 0.0), 1.0), I, 0, u, np.zeros((I, 3), np.float32))
    assert np.array_equal(cells, inner)
    cells, _ = G.sample(bits, res, 0, 0, ((0.0, 0.0, 0.0), 1.0), 0, I, u, np.zeros((I, 3), np.float32))
    want = np.nonzero(occ.reshape(-1) & G.interior(res, True))[0]
    assert set(cells.tolist()) == set(want.tolist())
    empty = O.pack_bits(np.zeros((res,) * 3, bool))
    cells, _ = G.sample(empty, res, 0, 0, ((0.0, 0.0, 0.0), 1.0), 0, I, u, np.zeros((I, 3), np.float32))
    assert np.array_equal(cells, inner)
