"""NumPy restatement of TSDF fusion (sparf_tsdf_integrate, include/sparf_b200.h) and of the masked marching cubes, plus
a PLY reader that takes uchar colour properties.

integrate: the header's rule taken literally, view after view.  The projection decides which pixel a point reads and
whether the view counts, so it is computed in fp32 with the header's op order (NumPy rounds each fp32 operation to
nearest, as the kernel's intrinsics do): the same views count for every point as in the kernel.  The running averages
(W tsdf + f) / (W + 1) and (W color + rgb) / (W + 1) are kept in fp64."""
import numpy as np

import mcubes_oracle as O

f32 = np.float32


def lattice_points(axis):
    """[n^3, 3] fp32, point (i, j, k) = (axis[i], axis[j], axis[k]) at linear index (i*n + j)*n + k"""
    a = np.asarray(axis, f32)
    return np.stack(np.meshgrid(a, a, a, indexing="ij"), -1).reshape(-1, 3)


def project(pts, pose, K):
    """camera coordinates x [P, 3] and pixel coordinates u, v [P] (fp32, the header's op order)"""
    x = [((pose[r, 0] * pts[:, 0] + pose[r, 1] * pts[:, 1]) + pose[r, 2] * pts[:, 2]) + pose[r, 3] for r in range(3)]
    with np.errstate(all="ignore"):
        u = ((K[0, 0] * x[0] + K[0, 1] * x[1]) + K[0, 2] * x[2]) / x[2]
        v = ((K[1, 0] * x[0] + K[1, 1] * x[1]) + K[1, 2] * x[2]) / x[2]
    return np.stack(x, 1), u, v


def integrate(axis, trunc, pose_w2c, intr, depth, rgb=None, valid=None, state=None):
    """-> (tsdf [n^3], weight [n^3], color [n^3, 3]) fp64 after the views of depth [B, H, W] in order, from `state`
    (the same triple) or the initial one (1, 0, 0)"""
    pts = lattice_points(axis)
    P = len(pts)
    if state is None:
        tsdf, weight, color = np.ones(P), np.zeros(P), np.zeros((P, 3))
    else:
        tsdf, weight, color = (np.array(s, np.float64) for s in state)
    pose_w2c, intr, depth = np.asarray(pose_w2c, f32), np.asarray(intr, f32), np.asarray(depth, f32)
    trunc = f32(trunc)
    B, H, W = depth.shape
    for b in range(B):
        x, u, v = project(pts, pose_w2c[b], intr[b] if intr.ndim == 3 else intr)
        with np.errstate(invalid="ignore"):
            ok = (x[:, 2] > 0) & (u >= 0) & (u < f32(W)) & (v >= 0) & (v < f32(H))
        idx = np.flatnonzero(ok)
        col, row = np.floor(u[idx]).astype(np.int64), np.floor(v[idx]).astype(np.int64)
        d = depth[b, row, col]
        keep = np.isfinite(d) & (d > 0)
        if valid is not None:
            keep &= np.asarray(valid)[b, row, col] != 0
        s = np.where(keep, d - x[idx, 2], f32(0))
        keep &= ~(s < -trunc)
        idx, row, col, s = idx[keep], row[keep], col[keep], s[keep]
        f = np.minimum(f32(1), s / trunc).astype(np.float64)
        w = weight[idx]
        tsdf[idx] = (w * tsdf[idx] + f) / (w + 1)
        if rgb is not None:
            color[idx] = (w[:, None] * color[idx] + np.asarray(rgb, f32)[b, row, col].astype(np.float64)) / (w[:, None] + 1)
        weight[idx] = w + 1
    return tsdf, weight, color


def masked_marching_cubes(vol, iso, table=None):
    """the dense mesh of mcubes_oracle.marching_cubes without the triangles of cells with a non-finite corner and
    without the vertices no remaining triangle uses, renumbered in their dense order"""
    table = O.case_table() if table is None else table
    vol = np.ascontiguousarray(vol, f32)
    verts, faces = O.marching_cubes(vol, iso, table)
    nx, ny, nz = vol.shape
    case = O.cell_cases(vol, iso).reshape(-1)
    ntri = (table >= 0).sum(1) // 3
    finite = np.ones((nx - 1, ny - 1, nz - 1), bool)
    fin = np.isfinite(vol)
    for di, dj, dk in O.CORNER_OFF:
        finite &= fin[di:nx - 1 + di, dj:ny - 1 + dj, dk:nz - 1 + dk]
    face_cell_ok = np.repeat(finite.reshape(-1), ntri[case])     # faces are cell-major, in table order within a cell
    assert len(face_cell_ok) == len(faces)
    faces = faces[face_cell_ok]
    used = np.zeros(len(verts), bool)
    used[faces.reshape(-1)] = True
    new_id = np.cumsum(used) - 1
    return verts[used], new_id[faces].reshape(-1, 3)


def read_ply(path):
    """binary little-endian PLY with float or uchar vertex properties and uchar-counted int face lists -> (header lines,
    structured vertex array, faces [F, 3] int64)"""
    with open(path, "rb") as f:
        data = f.read()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    header = data[:end].decode("ascii").splitlines()
    assert header[0] == "ply" and header[1] == "format binary_little_endian 1.0", header[:2]
    counts, props, cur = {}, [], None
    for line in header[2:]:
        w = line.split()
        if w[0] == "element":
            cur = w[1]
            counts[cur] = int(w[2])
        elif w[0] == "property" and cur == "vertex":
            props.append((w[2], {"float": "<f4", "uchar": "u1"}[w[1]]))
        elif w[0] == "property" and cur == "face":
            assert w[1:] == ["list", "uchar", "int", "vertex_indices"], line
    V, F = counts["vertex"], counts["face"]
    vert = np.frombuffer(data, np.dtype(props), V, end)
    face = np.frombuffer(data, np.dtype([("n", "u1"), ("v", "<i4", (3,))]), F, end + vert.nbytes)
    assert len(data) == end + vert.nbytes + face.nbytes and (face["n"] == 3).all()
    return header, vert.copy(), face["v"].astype(np.int64)
