"""NumPy restatement of the occupancy grid (include/sparf_b200.h, csrc/occupancy.cu): the bits built from a density
lattice, the per-sample lookup and the compaction.  Independent of the kernels: dilation by shifted maxima instead of a
per-cell window, the lookup vectorised over all samples, the compaction by np.nonzero."""
import numpy as np


def occupied_cells(sigma, thres):
    """bool [res]^3: cell c is occupied iff a lattice point with indices in [c-1, c+2] per axis has sigma >= thres or NaN"""
    sigma = np.asarray(sigma, np.float32)
    res = sigma.shape[0] - 1
    hot = ~(sigma < np.float32(thres))                     # >= thres, or NaN
    # a cell's own corners: lattice points c and c+1 per axis
    corner = np.zeros((res,) * 3, bool)
    for di in (0, 1):
        for dj in (0, 1):
            for dk in (0, 1):
                corner |= hot[di:di + res, dj:dj + res, dk:dk + res]
    # ... and those of its 26 neighbours: cells c-1 ... c+1 per axis, clipped
    out = np.zeros_like(corner)
    pad = np.pad(corner, 1)
    for di in range(3):
        for dj in range(3):
            for dk in range(3):
                out |= pad[di:di + res, dj:dj + res, dk:dk + res]
    return out


def pack_bits(occ):
    """bool [res]^3 -> uint32 words, cell idx = (i*res + j)*res + k at bit idx & 31 of word idx >> 5"""
    flat = np.asarray(occ, bool).reshape(-1)
    nw = (flat.size + 31) // 32
    padded = np.zeros(nw * 32, bool)
    padded[:flat.size] = flat
    weights = (np.uint64(1) << np.arange(32, dtype=np.uint64)).astype(np.uint64)
    return (padded.reshape(nw, 32).astype(np.uint64) * weights).sum(1).astype(np.uint32)


def unpack_bits(bits, res):
    bits = np.asarray(bits).view(np.uint32)
    idx = np.arange(res ** 3)
    return ((bits[idx >> 5] >> (idx & 31).astype(np.uint32)) & 1).astype(bool).reshape(res, res, res)


def build(sigma, thres):
    """the bitfield sparf_occupancy_build writes"""
    return pack_bits(occupied_cells(sigma, thres))


def kept(bits, res, r0, r1, origins, dirs, t):
    """bool [R,S]: sample x = o + t d (fp32, the MLP encoder's op order) is evaluated: outside the box (a u NaN, < 0 or
    >= res) or in an occupied cell"""
    f = np.float32
    o, d, t = np.asarray(origins, f), np.asarray(dirs, f), np.asarray(t, f)
    occ = unpack_bits(bits, res)
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        x = o[:, None, :] + d[:, None, :] * t[:, :, None]                        # each op rounds to fp32
        u = (x - f(r0)) / (f(r1) - f(r0)) * f(res)
        inside = ((u >= 0) & (u < f(res))).all(-1)
        cell = np.where(inside[..., None], u, 0).astype(np.int64)
    return ~inside | occ[cell[..., 0], cell[..., 1], cell[..., 2]]


def compact(bits, res, r0, r1, origins, dirs, t):
    """what sparf_occupancy_count/emit produce: (sample_idx [K] int64, origins_k [K,3], dirs_k [K,3], t_k [K,1])"""
    o, d, t = np.asarray(origins, np.float32), np.asarray(dirs, np.float32), np.asarray(t, np.float32)
    S = t.shape[1]
    idx = np.nonzero(kept(bits, res, r0, r1, o, d, t).reshape(-1))[0].astype(np.int64)
    r = idx // S
    return idx, o[r], d[r], t.reshape(-1)[idx][:, None]
