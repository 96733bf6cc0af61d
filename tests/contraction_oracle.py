"""NumPy restatement of the contracted occupancy grid (include/sparf_b200.h, csrc/compaction.cuh ContractedLookup,
sparf_b200/occupancy.py): the per-sample lookup in fp32 with every op rounded, the lattice of the build and its map to
world points, the exact (fp64) map and its inverse, and the compaction of one window.  The bits come from
occupancy_oracle.build; only the lookup and the lattice differ from the box grid."""
import numpy as np

import occupancy_oracle as O

f32 = np.float32


def contract_u(origins, dirs, t, center, radius, res):
    """u [R,S,3] fp32: x = o + d t, y = (x - c) / radius, m = max |y|, v = y (m <= 1) or y q (2 - q) with q = 1 / m,
    u = (v + 2) * 0.25 * res; each op rounded to fp32 (NumPy does not contract into FMAs)"""
    o, d, t = np.asarray(origins, f32), np.asarray(dirs, f32), np.asarray(t, f32)
    c = np.asarray(center, f32)
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        x = o[:, None, :] + d[:, None, :] * t[:, :, None]
        y = (x - c) / f32(radius)
        m = np.abs(y).max(-1, keepdims=True)                       # NaN if any |y| is NaN
        q = f32(1) / m
        v = np.where(m <= f32(1), y, (y * q) * (f32(2) - q))
        return ((v + f32(2)) * f32(0.25)) * f32(res)


def kept(bits, res, center, radius, origins, dirs, t):
    """bool [R,S]: the sample is evaluated: a u NaN or outside [0, res), or an occupied cell"""
    u = contract_u(origins, dirs, t, center, radius, res)
    occ = O.unpack_bits(bits, res)
    with np.errstate(invalid="ignore"):
        inside = ((u >= 0) & (u < f32(res))).all(-1)
        cell = np.where(inside[..., None], u, 0).astype(np.int64)
    return ~inside | occ[cell[..., 0], cell[..., 1], cell[..., 2]]


def compact(origins, dirs, t, k0, k1, alive, grid):
    """what sparf_contracted_count/emit produce for the window [k0, k1): (sample_idx [K] int64, origins_k [K,3],
    dirs_k [K,3], t_k [K,1]); grid = (bits, res, center, radius); alive None = every ray"""
    o, d, t = np.asarray(origins, f32), np.asarray(dirs, f32), np.asarray(t, f32)
    R, S = t.shape
    sel = np.zeros((R, S), bool)
    sel[:, k0:k1] = True
    if alive is not None:
        sel &= (np.asarray(alive) != 0)[:, None]
    sel &= kept(*grid, o, d, t)
    idx = np.nonzero(sel.reshape(-1))[0].astype(np.int64)
    r = idx // S
    return idx, o[r], d[r], t.reshape(-1)[idx][:, None]


# ------------------------------------------------------------------------------------------------ exact map (fp64)
def contract64(y):
    """the contraction of y = (x - c) / radius in fp64: y (||y||_inf <= 1) or y / m (2 - 1 / m)"""
    y = np.asarray(y, np.float64)
    m = np.abs(y).max(-1, keepdims=True)
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(m <= 1, y, y / m * (2 - 1 / m))


def uncontract64(v):
    """the inverse on ||v||_inf < 2: v (n <= 1) or v / (n (2 - n)), n = ||v||_inf"""
    v = np.asarray(v, np.float64)
    n = np.abs(v).max(-1, keepdims=True)
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(n <= 1, v, v / (n * (2 - n)))


# ------------------------------------------------------------------------------------------------ the build's lattice
def lattice_world(axis, center, radius):
    """(world points [n,n,n,3] fp32, far [n,n,n] bool) of the contracted lattice stack(meshgrid(axis, axis, axis)):
    center + radius * uncontract64(v) in fp64, rounded once to fp32; far = ||v||_inf >= 2 (at infinity, not evaluated;
    those points get the center)"""
    a = np.asarray(axis, f32).astype(np.float64)
    v = np.stack(np.meshgrid(a, a, a, indexing="ij"), -1)
    n = np.abs(v).max(-1, keepdims=True)
    far = n[..., 0] >= 2
    den = np.where((n <= 1) | far[..., None], 1.0, n * (2 - n))
    c = np.asarray(center, f32).astype(np.float64)
    x = np.where(far[..., None], c, c + float(f32(radius)) * (v / den))
    return x.astype(f32), far


def build(axis, center, radius, sigma_fn, thres):
    """the bits of a contracted grid whose density is sigma_fn(world points [..., 3] fp32) -> σ: NaN at infinity, then
    the box grid's build (dilation 1, NaN occupied)"""
    x, far = lattice_world(axis, center, radius)
    sigma = np.asarray(sigma_fn(x), f32)
    sigma = np.where(far, f32(np.nan), sigma)
    return O.build(sigma, thres)


def shell(res):
    """bool [res]^3: the outer two-cell shell (a cell index 0, 1, res-2 or res-1 on some axis)"""
    i = np.arange(res)
    edge = (i <= 1) | (i >= res - 2)
    return edge[:, None, None] | edge[None, :, None] | edge[None, None, :]
