"""NumPy reference of the ray cast of csrc/mesh_raycast.cu (include/sparf_b200.h, mesh ray cast): a vectorised brute
force of the same watertight ray/triangle test (Woop, Benthin and Wald, JCGT 2013) in fp64, and the same minimum of
(t, id) over every triangle with t in [t_min, t_max], ties to the smallest id.  Misses are inf / -1 / NaN."""
import numpy as np


def ray_triangles(o, d, a, b, c):
    """(t, bary [..., 3]) of the rays o + t d against the triangles abc (broadcast [..., 3], fp64): the two-sided
    watertight hit, t = inf and bary = NaN where there is none (edge functions of mixed sign, det = 0, zero area, or a
    ray with a non-finite component or d = 0)"""
    o, d, a, b, c = np.broadcast_arrays(*(np.asarray(x, np.float64) for x in (o, d, a, b, c)))
    k = np.argmax(np.abs(d), axis=-1)           # the first axis on ties, as the kernel
    kx, ky = (k + 1) % 3, (k + 2) % 3
    take = lambda v, i: np.take_along_axis(v, i[..., None], -1)[..., 0]
    dk = take(d, k)
    with np.errstate(all="ignore"):
        sx, sy, sz = take(d, kx) / dk, take(d, ky) / dk, 1.0 / dk

        def shear(v):
            A = v - o
            az = take(A, k)
            return take(A, kx) - sx * az, take(A, ky) - sy * az, sz * az

        (ax, ay, az), (bx, by, bz), (cx, cy, cz) = shear(a), shear(b), shear(c)
        U, V, W = cx * by - cy * bx, ax * cy - ay * cx, bx * ay - by * ax
        det = U + V + W
        t = (U * az + V * bz + W * cz) / det
        bary = np.stack([U, V, W], -1) / det[..., None]
        n = np.cross(b - a, c - a)
        ok = (np.isfinite(o).all(-1) & np.isfinite(d).all(-1) & (dk != 0) & (det != 0) & (n != 0).any(-1)
              & (((U >= 0) & (V >= 0) & (W >= 0)) | ((U <= 0) & (V <= 0) & (W <= 0))))
    return np.where(ok, t, np.inf), np.where(ok[..., None], bary, np.nan)


def raycast(origins, dirs, vertices, faces, t_min=0.0, t_max=np.inf, chunk=1 << 21):
    """(t [N], face [N] int64, bary [N, 3]): the brute-force first hit of every ray over every triangle (faces with ids
    outside [0, V) are never hit), ties to the smallest id (argmin's first)"""
    origins, dirs = np.asarray(origins, np.float64), np.asarray(dirs, np.float64)
    vertices = np.asarray(vertices, np.float64)
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    N = len(origins)
    t_out, f_out, b_out = np.full(N, np.inf), np.full(N, -1, np.int64), np.full((N, 3), np.nan)
    valid = ((faces >= 0) & (faces < len(vertices))).all(1)
    ids = np.nonzero(valid)[0]
    if len(ids) == 0 or N == 0:
        return t_out, f_out, b_out
    tri = vertices[faces[ids]]
    a, b, c = (tri[None, :, j] for j in range(3))
    rows = max(1, chunk // len(ids))
    for i0 in range(0, N, rows):
        o, d = origins[i0:i0 + rows, None], dirs[i0:i0 + rows, None]
        t, bary = ray_triangles(o, d, a, b, c)
        t = np.where((t >= t_min) & (t <= t_max), t, np.inf)
        j = np.argmin(t, axis=1)
        r = np.arange(len(j))
        hit = np.isfinite(t[r, j])
        t_out[i0:i0 + rows] = np.where(hit, t[r, j], np.inf)
        f_out[i0:i0 + rows] = np.where(hit, ids[j], -1)
        b_out[i0:i0 + rows] = np.where(hit[:, None], bary[r, j], np.nan)
    return t_out, f_out, b_out


def face_t(origins, dirs, vertices, faces, ids):
    """(t [N], bary [N, 3]) of ray i against face ids[i] alone (inf / NaN where it misses it)"""
    f = np.asarray(faces, np.int64)[ids]
    v = np.asarray(vertices, np.float64)
    return ray_triangles(origins, dirs, v[f[:, 0]], v[f[:, 1]], v[f[:, 2]])


def moller_trumbore(origins, dirs, vertices, faces, t_min=0.0, t_max=np.inf):
    """(t [N], face [N]): an independent two-sided Moller-Trumbore brute force in fp64 (no watertightness: a ray exactly
    through an edge may be counted in either, both or neither triangle)"""
    o = np.asarray(origins, np.float64)[:, None]
    d = np.asarray(dirs, np.float64)[:, None]
    v = np.asarray(vertices, np.float64)
    f = np.asarray(faces, np.int64)
    a, b, c = v[f[:, 0]][None], v[f[:, 1]][None], v[f[:, 2]][None]
    e1, e2 = b - a, c - a
    p = np.cross(d, e2)
    det = (e1 * p).sum(-1)
    with np.errstate(divide="ignore", invalid="ignore"):
        inv = 1.0 / det
        s = o - a
        u = (s * p).sum(-1) * inv
        q = np.cross(s, e1)
        w = (d * q).sum(-1) * inv
        t = (e2 * q).sum(-1) * inv
    ok = (det != 0) & (u >= 0) & (w >= 0) & (u + w <= 1) & (t >= t_min) & (t <= t_max)
    t = np.where(ok, t, np.inf)
    j = np.argmin(t, axis=1)
    r = np.arange(len(j))
    return t[r, j], np.where(np.isfinite(t[r, j]), j, -1)
