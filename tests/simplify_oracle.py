"""NumPy restatement of sparf_mesh_simplify (include/sparf_b200.h, mesh simplification): quadric-error edge collapses in
parallel rounds, run here one round at a time and one edge at a time.

Every fp64 step is a Python float operation, which rounds on its own like the device's __dadd_rn / __dmul_rn /
__ddiv_rn / __dsqrt_rn, in the device's order; fp32 roundings go through np.float32.  So the output equals the
device's bit for bit.  Fast enough for meshes of a few thousand faces.
"""
import math

import numpy as np


def f32(x):
    return float(np.float32(x))


def cross(p0, p1, p2):
    """(p1 - p0) x (p2 - p0)"""
    ux, uy, uz = p1[0] - p0[0], p1[1] - p0[1], p1[2] - p0[2]
    wx, wy, wz = p2[0] - p0[0], p2[1] - p0[1], p2[2] - p0[2]
    return (uy * wz - uz * wy, uz * wx - ux * wz, ux * wy - uy * wx)


def dot(a, b):
    return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]


def sub(a, b):
    return (a[0] - b[0], a[1] - b[1], a[2] - b[2])


def face_quadric(p0, p1, p2):
    """q_ij = (w n4_i) n4_j, ij = 00 01 02 03 11 12 13 22 23 33; n4 = (c / |c|, -n.p0), w = |c| / 2; 0 for |c| = 0"""
    c = cross(p0, p1, p2)
    ln = math.sqrt(dot(c, c))
    if not ln > 0.0:
        return [0.0] * 10
    n = (c[0] / ln, c[1] / ln, c[2] / ln)
    n4 = (n[0], n[1], n[2], -dot(n, p0))
    w = ln * 0.5
    return [(w * n4[i]) * n4[j] for i in range(4) for j in range(i, 4)]


def quad_eval(q, v):
    x, y, z = v
    r = (q[0] * x) * x
    r = r + 2.0 * ((q[1] * x) * y)
    r = r + 2.0 * ((q[2] * x) * z)
    r = r + 2.0 * (q[3] * x)
    r = r + (q[4] * y) * y
    r = r + 2.0 * ((q[5] * y) * z)
    r = r + 2.0 * (q[6] * y)
    r = r + (q[7] * z) * z
    r = r + 2.0 * (q[8] * z)
    return r + q[9]


def det3(a00, a01, a02, a10, a11, a12, a20, a21, a22):
    return (a00 * (a11 * a22 - a12 * a21) - a01 * (a10 * a22 - a12 * a20)) + a02 * (a10 * a21 - a11 * a20)


def place(pos, Q, bnd, a, b):
    """(v*, cost, survivor) of the edge (a, b), a < b"""
    q = [Q[a][i] + Q[b][i] for i in range(10)]
    pa, pb = pos[a], pos[b]
    if bnd[a] or bnd[b]:
        s = a if bnd[a] else b
        v = pos[s]
        return v, quad_eval(q, v), s
    det = det3(q[0], q[1], q[2], q[1], q[4], q[5], q[2], q[5], q[7])
    tr = (q[0] + q[4]) + q[7]
    if abs(det) > 1e-10 * ((tr * tr) * tr):
        b0, b1, b2 = -q[3], -q[6], -q[8]
        x = (f32(det3(b0, q[1], q[2], b1, q[4], q[5], b2, q[5], q[7]) / det),
             f32(det3(q[0], b0, q[2], q[1], b1, q[5], q[2], b2, q[7]) / det),
             f32(det3(q[0], q[1], b0, q[1], q[4], b1, q[2], q[5], b2) / det))
        mid = tuple((pa[i] + pb[i]) * 0.5 for i in range(3))
        dm, ab = sub(x, mid), sub(pb, pa)
        if dot(dm, dm) <= dot(ab, ab):
            return x, quad_eval(q, x), a
    mid = tuple(f32((pa[i] + pb[i]) * 0.5) for i in range(3))
    best = (pa, quad_eval(q, pa), a)
    cb, cm = quad_eval(q, pb), quad_eval(q, mid)
    if cb < best[1]:
        best = (pb, cb, a)
    if cm < best[1]:
        best = (mid, cm, a)
    return best


def third(f, a, b):
    return [x for x in f if x != a and x != b][0]


def link_ok(faces, vf, a, b, c, d):
    if c == d:
        return False
    nb_b = {x for i in vf[b] for x in faces[i]}
    for i in vf[a]:
        for x in faces[i]:
            if x not in (a, b, c, d) and x in nb_b:
                return False
    acd = any(c in faces[i] and d in faces[i] for i in vf[a])
    bcd = any(c in faces[i] and d in faces[i] for i in vf[b])
    return not (acd and bcd)


def no_fold(pos, faces, vf, v, a, b, vs):
    for i in vf[v]:
        f = faces[i]
        if a in f and b in f:
            continue
        p = [pos[x] for x in f]
        old = cross(*p)
        if old == (0.0, 0.0, 0.0):
            continue
        new = cross(*[vs if x == v else p[j] for j, x in enumerate(f)])
        if not dot(new, old) > 0.0:
            return False
    return True


def classify(pos, Q, faces):
    """-> (edges (sorted unique (lo, hi)), faces of each edge, faces of each vertex, boundary flags, valid keys)"""
    V = len(pos)
    edge_faces = {}
    vf = [[] for _ in range(V)]
    lock, bnd = [False] * V, [False] * V
    for i, f in enumerate(faces):
        for c in range(3):
            u, w = f[c], f[(c + 1) % 3]
            edge_faces.setdefault((min(u, w), max(u, w)), []).append(i)
            vf[u].append(i)
        if len(set(f)) < 3:
            for x in f:
                lock[x] = True
    edges = sorted(edge_faces)
    for (a, b) in edges:
        n = len(edge_faces[(a, b)])
        if n == 1:
            bnd[a] = bnd[b] = True
        elif n >= 3:
            lock[a] = lock[b] = True
    keys = []
    for e, (a, b) in enumerate(edges):
        ef = edge_faces[(a, b)]
        if len(ef) != 2 or lock[a] or lock[b] or (bnd[a] and bnd[b]):
            continue
        c, d = third(faces[ef[0]], a, b), third(faces[ef[1]], a, b)
        if not link_ok(faces, vf, a, b, c, d):
            continue
        v, cost, _ = place(pos, Q, bnd, a, b)
        if not (no_fold(pos, faces, vf, a, a, b, v) and no_fold(pos, faces, vf, b, a, b, v)):
            continue
        bits = int(np.float32(cost if cost > 0.0 else 0.0).view(np.uint32))
        keys.append(bits << 32 | e)
    return edges, edge_faces, vf, bnd, keys


def one_round(pos, Q, attrs, faces, target):
    """One round over the live faces (a list of id triples), in place on pos / Q / attrs -> (faces, removed ids)"""
    k = (len(faces) - target + 1) // 2
    edges, edge_faces, vf, bnd, keys = classify(pos, Q, faces)
    cands = sorted(keys)[:k]
    claim = {}
    for key in cands:
        a, b = edges[key & 0xffffffff]
        for x in {x for t in (a, b) for i in vf[t] for x in faces[i]}:
            claim[x] = min(claim.get(x, key), key)
    dead, ren = set(), {}
    for key in cands:
        a, b = edges[key & 0xffffffff]
        if any(claim[x] != key for t in (a, b) for i in vf[t] for x in faces[i]):
            continue
        v, _, s = place(pos, Q, bnd, a, b)
        r = b if s == a else a
        pa, pb = pos[a], pos[b]
        ab = sub(pb, pa)
        den = dot(ab, ab)
        t = dot(sub(v, pa), ab) / den if den > 0.0 else 0.0
        t = 0.0 if t < 0.0 else 1.0 if t > 1.0 else t
        if attrs is not None:
            xa, xb = attrs[a].astype(np.float64), attrs[b].astype(np.float64)
            attrs[s] = [f32(xa[j] + t * (xb[j] - xa[j])) for j in range(attrs.shape[1])]
        Q[s] = [Q[s][i] + Q[r][i] for i in range(10)]
        pos[s] = v
        ren[r] = s
        dead.update(edge_faces[(a, b)])
    faces = [tuple(ren.get(x, x) for x in f) for i, f in enumerate(faces) if i not in dead]
    return faces, list(ren)


def setup(vertices, faces):
    """-> (positions, quadrics, faces) as Python lists"""
    pos = [tuple(float(x) for x in p) for p in np.asarray(vertices, dtype=np.float32)]
    flist = [tuple(int(x) for x in f) for f in np.asarray(faces, dtype=np.int64).reshape(-1, 3)]
    Q = [[0.0] * 10 for _ in range(len(pos))]
    for f in flist:
        fq = face_quadric(*[pos[x] for x in f])
        for x in f:
            Q[x] = [Q[x][i] + fq[i] for i in range(10)]
    return pos, Q, flist


def simplify(vertices, faces, target, attrs=None):
    """-> (vertices [V', 3] fp32, faces [F', 3] int64, vert_ids [V'] int64, attrs [V', A] fp32 or None, rounds)"""
    pos, Q, flist = setup(vertices, faces)
    attrs = None if attrs is None else np.array(attrs, dtype=np.float32)
    V = len(pos)
    removed = np.zeros(V, dtype=bool)
    rounds = 0
    while len(flist) > target:
        flist, gone = one_round(pos, Q, attrs, flist, target)
        rounds += 1
        if not gone:
            break
        removed[gone] = True
    keep = np.flatnonzero(~removed)
    new_id = np.full(V, -1, dtype=np.int64)
    new_id[keep] = np.arange(keep.size)
    out_v = np.array([pos[i] for i in keep], dtype=np.float32).reshape(-1, 3)
    out_f = new_id[np.array(flist, dtype=np.int64).reshape(-1, 3)] if flist else np.zeros((0, 3), np.int64)
    out_a = None if attrs is None else attrs[keep]
    return out_v, out_f, keep.astype(np.int64), out_a, rounds
