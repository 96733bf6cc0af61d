"""NumPy restatement of sparse marching cubes (include/sparf_b200.h, "sparse marching cubes"), built on mcubes_oracle.

classify() applies the block rule to a coarse lattice.  marching_cubes_blocks() works from what the kernels see, the
σ of each active block and the block ids: it meshes every block on its own with the dense oracle, names each vertex by
its global key (linear p) * 3 + a, merges the blocks' vertices by key and orders the triangles by global cell.
dense_filtered() is the specification's other side: the dense oracle's mesh without the triangles of inactive blocks
and without the vertices no remaining triangle uses."""
import numpy as np

import mcubes_oracle as O

B = 8


def classify(coarse, iso):
    """coarse [nb+1]^3 -> active [nb, nb, nb] bool: the window [b-1, b+2] per axis (clipped to [0, nb]) holds a NaN, or
    a value >= iso and a value < iso"""
    c = np.asarray(coarse, np.float32)
    nb = c.shape[0] - 1
    nan = np.isnan(c)
    with np.errstate(invalid="ignore"):
        ins, outs = (c >= np.float32(iso)) & ~nan, (c < np.float32(iso)) & ~nan
    active = np.zeros((nb, nb, nb), bool)
    for bi in range(nb):
        for bj in range(nb):
            for bk in range(nb):
                w = tuple(slice(max(x - 1, 0), min(x + 2, nb) + 1) for x in (bi, bj, bk))
                active[bi, bj, bk] = nan[w].any() or (ins[w].any() and outs[w].any())
    return active


def block_points(vol, block_ids, nb):
    """sigma [n, 9, 9, 9] of the given blocks cut from a full [8 nb + 1]^3 volume"""
    out = np.empty((len(block_ids), B + 1, B + 1, B + 1), np.float32)
    for r, b in enumerate(block_ids):
        bi, bj, bk = np.unravel_index(int(b), (nb, nb, nb))
        out[r] = vol[B * bi:B * bi + B + 1, B * bj:B * bj + B + 1, B * bk:B * bk + B + 1]
    return out


def _cell_of_faces(vol, iso, table):
    """the linear cell index of each face of the dense oracle's mesh of vol (cells in order, table rows in order)"""
    case = O.cell_cases(vol, iso).reshape(-1)
    ntri = (table >= 0).sum(1) // 3
    return np.repeat(np.arange(case.size), ntri[case])


def dense_filtered(vol, iso, active, table=None):
    """the dense oracle's mesh of vol [8 nb + 1]^3 with only the triangles of cells in active blocks, the unused vertices
    dropped and the rest renumbered in order"""
    table = O.case_table() if table is None else table
    vol = np.ascontiguousarray(vol, np.float32)
    verts, faces = O.marching_cubes(vol, iso, table)
    n = vol.shape[0] - 1
    ci, cj, ck = np.unravel_index(_cell_of_faces(vol, iso, table), (n, n, n))
    faces = faces[active[ci // B, cj // B, ck // B]]
    used = np.unique(faces)
    remap = np.full(len(verts), -1, np.int64)
    remap[used] = np.arange(len(used))
    return verts[used], remap[faces]


def marching_cubes_blocks(sigma_blocks, block_ids, res, iso, table=None):
    """(verts [V, 3] fp32, faces [F, 3] int64) in index space from the σ [n, 9, 9, 9] of the active blocks block_ids"""
    table = O.case_table() if table is None else table
    iso = np.float32(iso)
    nb, n = res // B, res + 1
    keys, pos, fkeys, fcell = [], [], [], []
    for r, b in enumerate(block_ids):
        blk = np.array(np.unravel_index(int(b), (nb, nb, nb))) * B
        sig = np.ascontiguousarray(sigma_blocks[r], np.float32)
        _, lf = O.marching_cubes(sig, iso, table)
        # the block's vertex keys in the dense oracle's (local p, a) order
        with np.errstate(invalid="ignore"):
            inside = sig >= iso
        cross = np.zeros(sig.shape + (3,), bool)
        cross[:-1, :, :, 0] = inside[:-1] != inside[1:]
        cross[:, :-1, :, 1] = inside[:, :-1] != inside[:, 1:]
        cross[:, :, :-1, 2] = inside[:, :, :-1] != inside[:, :, 1:]
        q = np.flatnonzero(cross.reshape(-1))
        lp, a = q // 3, q % 3
        p = np.stack(np.unravel_index(lp, sig.shape), 1) + blk
        k = ((p[:, 0] * n + p[:, 1]) * n + p[:, 2]) * 3 + a
        # positions as the dense extractor computes them: float(p_a) + (iso - v0) / (v1 - v0) in fp32
        off = np.eye(3, dtype=np.int64)[a]
        lq = np.stack(np.unravel_index(lp, sig.shape), 1)
        v0 = sig[lq[:, 0], lq[:, 1], lq[:, 2]]
        v1 = sig[lq[:, 0] + off[:, 0], lq[:, 1] + off[:, 1], lq[:, 2] + off[:, 2]]
        with np.errstate(all="ignore"):
            s = (iso - v0) / (v1 - v0)
        xyz = p.astype(np.float32)
        rows = np.arange(len(q))
        xyz[rows, a] = xyz[rows, a] + s
        keys.append(k)
        pos.append(xyz)
        fkeys.append(k[lf])
        lc = np.stack(np.unravel_index(_cell_of_faces(sig, iso, table), (B, B, B)), 1) + blk
        fcell.append((lc[:, 0] * res + lc[:, 1]) * res + lc[:, 2])
    if not keys:
        return np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int64)
    keys, pos = np.concatenate(keys), np.concatenate(pos)
    uk, first = np.unique(keys, return_index=True)
    verts = pos[first]
    fkeys, fcell = np.concatenate(fkeys), np.concatenate(fcell)
    order = np.argsort(fcell, kind="stable")        # cells are disjoint between blocks: table order kept per cell
    faces = np.searchsorted(uk, fkeys[order])
    return verts, faces.astype(np.int64)
