"""From-scratch, vectorised NumPy restatement of the marching cubes that include/sparf_b200.h specifies
(sparf_mcubes_count / sparf_mcubes_emit), plus mesh checks and a binary PLY reader for the tests.

The oracle reads only the case table from the library (sparf_mcubes_table); inside test, vertex ownership, ordering,
interpolation and the edge-to-vertex mapping are restated here.  Its vertices are the kernels' bit for bit (the same
fp32 operations in the same order) and its faces equal theirs."""
import numpy as np

# edge e = 4a + m: along axis a from the cell corner whose offsets along the two other axes b < b' are (m & 1, m >> 1)
EDGE_AXIS = np.array([e // 4 for e in range(12)])
EDGE_OFF = np.zeros((12, 3), np.int64)
for _e in range(12):
    _b, _b2 = [x for x in range(3) if x != _e // 4]
    EDGE_OFF[_e, _b], EDGE_OFF[_e, _b2] = _e % 4 & 1, _e % 4 >> 1
# corner c of a cell at offset (c & 1, (c >> 1) & 1, (c >> 2) & 1)
CORNER_OFF = np.array([[c & 1, (c >> 1) & 1, (c >> 2) & 1] for c in range(8)])


def case_table():
    """[256, 3 * MCUBES_MAX_TRIS] int8, the library's table (edge ids, -1 padded)"""
    from sparf_b200 import _lib
    t = np.empty((256, 3 * _lib.MCUBES_MAX_TRIS), np.int8)
    _lib.check(_lib.lib().sparf_mcubes_table(t.ctypes.data), "mcubes_table")
    return t


def crossing_edges(case):
    """cell-edge ids whose two corners differ in case `case`"""
    out = []
    for e in range(12):
        c0 = EDGE_OFF[e]
        c1 = c0.copy()
        c1[EDGE_AXIS[e]] = 1
        b0 = (case >> int(c0[0] | c0[1] << 1 | c0[2] << 2)) & 1
        b1 = (case >> int(c1[0] | c1[1] << 1 | c1[2] << 2)) & 1
        if b0 != b1:
            out.append(e)
    return out


def cell_cases(vol, iso):
    """case index of every cell, [nx-1, ny-1, nz-1]"""
    with np.errstate(invalid="ignore"):
        inside = (np.asarray(vol, np.float32) >= np.float32(iso)).astype(np.int32)
    nx, ny, nz = inside.shape
    case = np.zeros((nx - 1, ny - 1, nz - 1), np.int32)
    for c, (di, dj, dk) in enumerate(CORNER_OFF):
        case |= inside[di:nx - 1 + di, dj:ny - 1 + dj, dk:nz - 1 + dk] << c
    return case


def marching_cubes(vol, iso, table=None):
    """vol [nx, ny, nz] fp32, iso -> (verts [V, 3] fp32, faces [F, 3] int64) in index space"""
    table = case_table() if table is None else table
    vol = np.ascontiguousarray(vol, dtype=np.float32)
    iso = np.float32(iso)
    nx, ny, nz = vol.shape
    assert min(vol.shape) >= 2
    with np.errstate(invalid="ignore"):
        inside = vol >= iso                       # NaN: outside
    cross = np.zeros(vol.shape + (3,), bool)      # cross[p, a]: the lattice edge p -> p + e_a crosses
    cross[:-1, :, :, 0] = inside[:-1] != inside[1:]
    cross[:, :-1, :, 1] = inside[:, :-1] != inside[:, 1:]
    cross[:, :, :-1, 2] = inside[:, :, :-1] != inside[:, :, 1:]
    flat = cross.reshape(-1)
    vid = np.cumsum(flat, dtype=np.int64) - 1     # vertex id of (p, a), ordered by (linear p, a)
    q = np.flatnonzero(flat)
    p, a = q // 3, q % 3
    strides = np.array([ny * nz, nz, 1], np.int64)
    v0 = vol.reshape(-1)[p]
    v1 = vol.reshape(-1)[p + strides[a]]
    with np.errstate(all="ignore"):
        s = (iso - v0) / (v1 - v0)                # fp32, as written
    verts = np.stack(np.unravel_index(p, vol.shape), 1).astype(np.float32)
    rows = np.arange(len(q))
    verts[rows, a] = verts[rows, a] + s           # float(p_a) + s in fp32
    case = cell_cases(vol, iso).reshape(-1)
    cells = np.flatnonzero((case != 0) & (case != 255))   # linear cell order
    ci, cj, ck = np.unravel_index(cells, (nx - 1, ny - 1, nz - 1))
    tri = table[case[cells]].astype(np.int64)              # [C, 15]
    r, c = np.nonzero(tri >= 0)                            # cell-major, table order within a cell
    e = tri[r, c]
    oi, oj, ok = ci[r] + EDGE_OFF[e, 0], cj[r] + EDGE_OFF[e, 1], ck[r] + EDGE_OFF[e, 2]
    faces = vid[((oi * ny + oj) * nz + ok) * 3 + EDGE_AXIS[e]].reshape(-1, 3)
    return verts, faces


def directed_edges(faces):
    faces = np.asarray(faces, np.int64)
    return np.concatenate([faces[:, [0, 1]], faces[:, [1, 2]], faces[:, [2, 0]]])


def is_closed_and_oriented(faces):
    """every undirected edge lies in exactly two triangles, once in each direction"""
    d = directed_edges(faces)
    if len(d) == 0:
        return True
    n = int(d.max()) + 1
    key, rkey = d[:, 0] * n + d[:, 1], d[:, 1] * n + d[:, 0]
    return len(np.unique(key)) == len(key) and bool(np.isin(rkey, key).all())


def euler_characteristic(faces):
    faces = np.asarray(faces, np.int64)
    return len(np.unique(faces)) - len(directed_edges(faces)) // 2 + len(faces)


def face_normals(verts, faces):
    v = np.asarray(verts, np.float64)[np.asarray(faces)]
    return np.cross(v[:, 1] - v[:, 0], v[:, 2] - v[:, 0])


def read_ply(path):
    """binary little-endian PLY with float vertex properties and uchar-counted int face lists ->
    (dict name -> [V] float32 array, faces [F, 3] int64)"""
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
            assert w[1] == "float", line
            props.append(w[2])
        elif w[0] == "property" and cur == "face":
            assert w[1:] == ["list", "uchar", "int", "vertex_indices"], line
    V, F = counts["vertex"], counts["face"]
    vert = np.frombuffer(data, np.dtype([(p, "<f4") for p in props]), V, end)
    face = np.frombuffer(data, np.dtype([("n", "u1"), ("v", "<i4", (3,))]), F, end + vert.nbytes)
    assert len(data) == end + vert.nbytes + face.nbytes and (face["n"] == 3).all()
    return {p: vert[p].copy() for p in props}, face["v"].astype(np.int64)
