"""NumPy reference of the closest-point queries of csrc/mesh_distance.cu (include/sparf_b200.h, mesh distance): a
vectorised brute force, in fp64 unless the inputs are fp32.  Point to triangle by the kernel's case analysis: the
projection onto the plane when the normal is nonzero and the projection lies inside the triangle, else (and on ties
after it) the nearest of the clamped projections onto the edges ab, bc, ca.  Point to point by scipy's cKDTree."""
import numpy as np


def _dot(a, b):
    return (a * b).sum(-1)


def closest_on_segment(p, a, b):
    """the closest point of the segments a -> b to p (broadcast [..., 3]); parameter 0 where a = b"""
    ab = b - a
    l = _dot(ab, ab)
    t = np.where(l > 0, _dot(p - a, ab) / np.where(l > 0, l, 1), 0)
    return a + np.clip(t, 0, 1)[..., None] * ab


def closest_on_triangle(p, a, b, c):
    """(q [..., 3], d2 [...]): the closest point of triangles abc to p and its squared distance"""
    q = closest_on_segment(p, a, b)
    d2 = _dot(p - q, p - q)
    for u, v in ((b, c), (c, a)):
        qe = closest_on_segment(p, u, v)
        de = _dot(p - qe, p - qe)
        take = de < d2
        q, d2 = np.where(take[..., None], qe, q), np.where(take, de, d2)
    ab, ac, ap = b - a, c - a, p - a
    # fp32 inputs model the kernel, whose face normal is the nearly correctly rounded cross product
    n = np.cross(ab.astype(np.float64), ac.astype(np.float64)).astype(ab.dtype)
    nn = _dot(n, n)
    inside = ((nn > 0) & (_dot(n, np.cross(ab, ap)) >= 0) & (_dot(n, np.cross(c - b, p - b)) >= 0)
              & (_dot(n, np.cross(a - c, p - c)) >= 0))
    qf = p - (_dot(n, ap) / np.where(nn > 0, nn, 1))[..., None] * n
    df = _dot(p - qf, p - qf)
    take = inside & (df <= d2)
    return np.where(take[..., None], qf, q), np.where(take, df, d2)


def barycentric(q, a, b, c):
    """the barycentric coordinates [..., 3] of q in triangles abc (least squares; NaN for zero area)"""
    ab, ac, aq = b - a, c - a, q - a
    d00, d01, d11 = _dot(ab, ab), _dot(ab, ac), _dot(ac, ac)
    d20, d21 = _dot(aq, ab), _dot(aq, ac)
    den = d00 * d11 - d01 * d01
    with np.errstate(divide="ignore", invalid="ignore"):
        v = (d11 * d20 - d01 * d21) / den
        w = (d00 * d21 - d01 * d20) / den
    return np.stack([1 - v - w, v, w], -1)


def triangle_distance(points, vertices, faces, ids):
    """(d [N], q [N, 3]): the distance and closest point of triangle ids[i] to points[i]"""
    f = faces[ids]
    q, d2 = closest_on_triangle(points, vertices[f[:, 0]], vertices[f[:, 1]], vertices[f[:, 2]])
    return np.sqrt(d2), q


def closest_triangles(points, vertices, faces, max_dist=np.inf, chunk=1 << 22):
    """(dist [N], index [N] int64, closest [N, 3], d_all or None): the brute-force minimum over every triangle, ties to
    the smallest id (argmin's first); misses (nothing within max_dist, or no triangle) give inf / -1 / NaN"""
    points, vertices = np.asarray(points, np.float64), np.asarray(vertices, np.float64)
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    N, F = len(points), len(faces)
    dist, index, closest = np.full(N, np.inf), np.full(N, -1, np.int64), np.full((N, 3), np.nan)
    if F == 0 or N == 0:
        return dist, index, closest
    a, b, c = (vertices[faces[:, k]][None] for k in range(3))
    rows = max(1, chunk // F)
    for i0 in range(0, N, rows):
        p = points[i0:i0 + rows, None]
        q, d2 = closest_on_triangle(p, a, b, c)
        k = np.argmin(d2, axis=1)
        r = np.arange(len(k))
        d = np.sqrt(d2[r, k])
        hit = d <= max_dist
        dist[i0:i0 + rows] = np.where(hit, d, np.inf)
        index[i0:i0 + rows] = np.where(hit, k, -1)
        closest[i0:i0 + rows] = np.where(hit[:, None], q[r, k], np.nan)
    return dist, index, closest


def closest_vertices(points, vertices, max_dist=np.inf):
    """(dist [N], index [N] int64, closest [N, 3]) against the point cloud vertices (cKDTree; among equal distances
    any id); misses give inf / -1 / NaN"""
    from scipy.spatial import cKDTree
    points, vertices = np.asarray(points, np.float64), np.asarray(vertices, np.float64)
    N = len(points)
    dist, index, closest = np.full(N, np.inf), np.full(N, -1, np.int64), np.full((N, 3), np.nan)
    if len(vertices) == 0 or N == 0:
        return dist, index, closest
    d, k = cKDTree(vertices).query(points, k=1)
    hit = d <= max_dist
    dist[hit], index[hit], closest[hit] = d[hit], k[hit], vertices[k[hit]]
    return dist, index, closest


def closest_triangles_near(points, vertices, faces, radius):
    """closest_triangles restricted to the triangles whose centroid lies within radius[i] + the largest
    centroid-to-vertex distance of point i: exact for every point whose nearest triangle lies within radius[i] (the
    rest get inf / -1 / NaN).  For meshes too large for the brute force."""
    from scipy.spatial import cKDTree
    points, vertices = np.asarray(points, np.float64), np.asarray(vertices, np.float64)
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    tri = vertices[faces]
    cen = tri.mean(1)
    reach = np.sqrt(((tri - cen[:, None]) ** 2).sum(-1)).max()
    tree = cKDTree(cen)
    N = len(points)
    dist, index, closest = np.full(N, np.inf), np.full(N, -1, np.int64), np.full((N, 3), np.nan)
    for i, cand in enumerate(tree.query_ball_point(points, np.asarray(radius) + reach)):
        if not cand:
            continue
        cand = np.sort(np.asarray(cand, np.int64))
        q, d2 = closest_on_triangle(points[i][None], tri[cand, 0], tri[cand, 1], tri[cand, 2])
        k = np.argmin(d2)
        if np.sqrt(d2[k]) <= radius[i]:
            dist[i], index[i], closest[i] = np.sqrt(d2[k]), cand[k], q[k]
    return dist, index, closest
