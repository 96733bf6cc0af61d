"""NumPy restatement of early ray termination (include/sparf_b200.h, csrc/termination.cu): the sequential fp32 optical
depth with each op rounded, the windowed mask of evaluated samples given the dense σ, and the compaction of one window,
with the occupancy lookup of occupancy_oracle.  Vectorised over the rays, sequential in k only."""
import math

import numpy as np

import occupancy_oracle as O

f32 = np.float32


def tau_max(eps):
    """fp32(-ln eps); eps = 0: +inf"""
    return f32(-math.log(eps)) if eps > 0 else f32(np.inf)


def ray_len(dirs):
    """sqrt((dx dx + dy dy) + dz dz), each op rounded to fp32"""
    d = np.asarray(dirs, f32)
    with np.errstate(over="ignore", invalid="ignore"):
        return np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])


def update(sigma, t, dirs, k0, k1, tmax, tau, alive):
    """what sparf_termination_update writes: (tau [R] float32, alive [R] uint8).  Rays with alive 0 are untouched."""
    sigma, t = np.asarray(sigma, f32), np.asarray(t, f32)
    S = t.shape[1]
    length = ray_len(dirs)
    alive = np.asarray(alive, np.uint8).copy()
    acc = np.asarray(tau, f32).copy()
    on = alive != 0
    with np.errstate(over="ignore", invalid="ignore"):
        for k in range(k0, k1):
            gap = t[:, k + 1] - t[:, k] if k + 1 < S else np.full(t.shape[0], 1e10, f32)
            acc = np.where(on, acc + sigma[:, k] * (gap * length), acc).astype(f32)
        alive[on & (acc > f32(tmax))] = 0
    return acc, alive


def evaluated(sigma, t, dirs, eps, window, keep=None):
    """bool [R,S]: the samples a termination render evaluates, given the dense σ [R,S] (only its evaluated samples
    matter) and the occupancy grid's kept mask (None = no grid)"""
    sigma, t = np.asarray(sigma, f32), np.asarray(t, f32)
    R, S = t.shape
    keep = np.ones((R, S), bool) if keep is None else np.asarray(keep, bool)
    ev = np.zeros((R, S), bool)
    alive, tau = np.ones(R, np.uint8), np.zeros(R, f32)
    tmax = tau_max(eps)
    for k0 in range(0, S, window):
        k1 = min(k0 + window, S)
        ev[:, k0:k1] = (alive != 0)[:, None] & keep[:, k0:k1]
        if k1 < S:
            tau, alive = update(np.where(ev, sigma, f32(0)), t, dirs, k0, k1, tmax, tau, alive)
    return ev


def compact(origins, dirs, t, k0, k1, alive=None, grid=None):
    """what sparf_termination_count/emit produce for the window [k0, k1): (sample_idx [K] int64, origins_k [K,3],
    dirs_k [K,3], t_k [K,1]); grid = (bits, res, r0, r1) or None"""
    o, d, t = np.asarray(origins, f32), np.asarray(dirs, f32), np.asarray(t, f32)
    R, S = t.shape
    sel = np.zeros((R, S), bool)
    sel[:, k0:k1] = True
    if alive is not None:
        sel &= (np.asarray(alive) != 0)[:, None]
    if grid is not None:
        sel &= O.kept(*grid, o, d, t)
    idx = np.nonzero(sel.reshape(-1))[0].astype(np.int64)
    r = idx // S
    return idx, o[r], d[r], t.reshape(-1)[idx][:, None]
