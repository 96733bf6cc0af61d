"""NumPy restatement of the occupancy grid update (include/sparf_b200.h "occupancy grid update", csrc/grid_update.cu,
sparf_b200/occupancy.py update_): the interior cells, the sampled cells and their points in fp64 with every op rounded
(NumPy does not contract into FMAs), the decaying per-cell density and its threshold, and the corner max that
build_grid(ema=True) starts the density from."""
import numpy as np

import occupancy_oracle as O

f32 = np.float32
FLT_MAX = np.finfo(f32).max


def interior(res, contracted):
    """bool [res^3] by linear index: every cell of a box grid, the cells with every index in [2, res-3] of a contracted
    one"""
    if not contracted:
        return np.ones(res ** 3, bool)
    i = np.arange(res)
    m = (i >= 2) & (i <= res - 3)
    return (m[:, None, None] & m[None, :, None] & m[None, None, :]).reshape(-1)


def _pick(u, n):
    """min(floor((double)u * n), n - 1), clamped at 0"""
    j = np.floor(np.asarray(u, f32).astype(np.float64) * float(n)).astype(np.int64)
    return np.clip(j, 0, n - 1)


def sample(bits, res, r0, r1, contraction, n_uniform, n_occupied, u_cell, u_jit):
    """(cells [N] int64, points [N,3] fp32) of sparf_occupancy_sample; contraction None = a box grid over [r0, r1]^3,
    else (center, radius) as fp32 values"""
    contracted = contraction is not None
    inner = np.nonzero(interior(res, contracted))[0]
    occ = np.nonzero(O.unpack_bits(bits, res).reshape(-1) & interior(res, contracted))[0]
    u_cell = np.asarray(u_cell, f32)
    n = n_uniform + n_occupied
    cells = np.empty(n, np.int64)
    uniform = (np.arange(n) < n_uniform) | (occ.size == 0)
    cells[uniform] = inner[_pick(u_cell[uniform], inner.size)]
    if (~uniform).any():
        cells[~uniform] = occ[_pick(u_cell[~uniform], occ.size)]
    return cells, points(cells, res, r0, r1, contraction, u_jit)


def points(cells, res, r0, r1, contraction, u_jit):
    """the fp32 point of each sample in its cell (jitter u_jit [N,3])"""
    c = np.stack([cells // (res * res), cells // res % res, cells % res], -1).astype(np.float64)
    x = c + np.asarray(u_jit, f32).astype(np.float64)
    if contraction is None:
        a, b = float(f32(r0)), float(f32(r1))
        return (a + (x * (b - a)) / res).astype(f32)
    center, radius = contraction
    v = -2.0 + (x * 4.0) / res
    nrm = np.abs(v).max(-1, keepdims=True)
    den = np.where(nrm <= 1.0, 1.0, nrm * (2.0 - nrm))
    ctr = np.asarray(center, f32).astype(np.float64)
    return (ctr + float(f32(radius)) * (v / den)).astype(f32)


def ema(density, res, contracted, cells, sigma, decay, thres):
    """(density [res^3] fp32, bits) after sparf_occupancy_ema"""
    d = np.asarray(density, f32).copy()
    s = np.asarray(sigma, f32)
    with np.errstate(invalid="ignore"):
        s = np.where(np.isnan(s) | (s == np.inf), FLT_MAX, s)
    smax = np.zeros(res ** 3, f32)
    np.maximum.at(smax, np.asarray(cells, np.int64), s)
    inner = interior(res, contracted)
    d[inner] = np.maximum(f32(decay) * d[inner], smax[inner])
    with np.errstate(invalid="ignore"):
        occ = ~(d < f32(thres)) | ~inner
    return d, O.pack_bits(occ.reshape(res, res, res))


def corner_max(sigma):
    """lattice σ [res+1]^3 -> the per-cell density [res^3]: the max over each cell's 8 corners, NaN and +inf as FLT_MAX"""
    s = np.asarray(sigma, f32)
    s = np.where(np.isnan(s) | (s == np.inf), FLT_MAX, s)
    n = s.shape[0] - 1
    d = s[:n, :n, :n].copy()
    for a in (0, 1):
        for b in (0, 1):
            for c in (0, 1):
                d = np.maximum(d, s[a:a + n, b:b + n, c:c + n])
    return d.reshape(-1)
