#!/usr/bin/env python
"""Generate mcubes_table.cuh, the marching-cubes case table of csrc/mcubes.cu.

    python sparf_b200/csrc/mcubes_table.py        # rewrites mcubes_table.cuh next to this file

Conventions (include/sparf_b200.h, sparf_mcubes_table):
  corner c of a cell sits at offset (c & 1, (c >> 1) & 1, (c >> 2) & 1) along (i, j, k); the case index has bit c set
  when corner c is inside (vol >= iso).
  edge e = 4 a + m runs along axis a from the corner with offset 0 along a; its offsets along the two other axes
  b < b' are (m & 1, m >> 1).

The table is derived from one rule per cube face, so that two cells sharing a face cut it the same way:
  * a face with two crossing edges gets one segment between them;
  * a face with four (two inside corners on a diagonal) gets two segments, each cutting off one inside corner: inside
    corners never connect across a face, outside corners always do.
Each segment is directed so that (end - start) x (outward face normal) points to the inside side.  The directed
segments of a case form disjoint cycles; each cycle is triangulated in its own direction, so (v1 - v0) x (v2 - v0)
points from the inside toward the outside, with no diagonal between two edges of one cube face (an edge of a shared
face would then also be an edge of the neighbouring cell and could lie in more than two triangles).  A mesh built with
this table is closed and consistently oriented wherever no inside point lies on the volume's border.
"""
import os

AXES = range(3)
MAX_TRIS = 5        # SPARF_MCUBES_MAX_TRIS


def corner(off):
    return off[0] | off[1] << 1 | off[2] << 2


def offset(c):
    return (c & 1, (c >> 1) & 1, (c >> 2) & 1)


def others(a):
    return [b for b in AXES if b != a]


def edge_id(c0, c1):
    o0, o1 = offset(c0), offset(c1)
    (a,) = [x for x in AXES if o0[x] != o1[x]]
    lo = o0 if o0[a] == 0 else o1
    b, b2 = others(a)
    return 4 * a + (lo[b] | lo[b2] << 1)


def edge_mid(e):
    a, m = divmod(e, 4)
    b, b2 = others(a)
    p = [0.0, 0.0, 0.0]
    p[a], p[b], p[b2] = 0.5, float(m & 1), float(m >> 1)
    return p


def edge_faces(e):
    a, m = divmod(e, 4)
    b, b2 = others(a)
    return {(b, m & 1), (b2, m >> 1)}


def sub(x, y):
    return [u - v for u, v in zip(x, y)]


def cross(x, y):
    return [x[1] * y[2] - x[2] * y[1], x[2] * y[0] - x[0] * y[2], x[0] * y[1] - x[1] * y[0]]


def dot(x, y):
    return sum(u * v for u, v in zip(x, y))


def segments(case):
    """directed (edge, edge) segments of all six faces"""
    inside = [(case >> c) & 1 for c in range(8)]
    segs = []
    for a in AXES:
        b, b2 = others(a)
        for s in (0, 1):
            normal = [0.0, 0.0, 0.0]
            normal[a] = 1.0 if s else -1.0
            cyc = []
            for ob, ob2 in ((0, 0), (1, 0), (1, 1), (0, 1)):
                o = [0, 0, 0]
                o[a], o[b], o[b2] = s, ob, ob2
                cyc.append(corner(o))
            cuts = [q for q in range(4) if inside[cyc[q]] != inside[cyc[(q + 1) % 4]]]
            if len(cuts) == 2:      # one segment; any inside corner lies on its inside side
                pairs = [(cuts[0], cuts[1], next(c for c in cyc if inside[c]))]
            elif len(cuts) == 4:    # cut off each inside corner on its own
                pairs = [((q - 1) % 4, q, cyc[q]) for q in range(4) if inside[cyc[q]]]
            else:
                pairs = []
            for q0, q1, k in pairs:
                e0 = edge_id(cyc[q0], cyc[(q0 + 1) % 4])
                e1 = edge_id(cyc[q1], cyc[(q1 + 1) % 4])
                p0, p1 = edge_mid(e0), edge_mid(e1)
                mid = [(u + v) / 2 for u, v in zip(p0, p1)]
                if dot(cross(sub(p1, p0), normal), sub(list(map(float, offset(k))), mid)) < 0:
                    e0, e1 = e1, e0
                segs.append((e0, e1))
    return segs


def triangulate(poly):
    """triangles of the cycle `poly` in its direction, no diagonal joining two edges of one face; None if impossible"""
    n = len(poly)
    if n == 3:
        return [tuple(poly)]
    ok = lambda u, v: not (edge_faces(u) & edge_faces(v))
    for k in range(2, n):
        if (k != 2 and not ok(poly[1], poly[k])) or (k != n - 1 and not ok(poly[k], poly[0])):
            continue
        left = triangulate(poly[1:k + 1]) if k > 2 else []
        right = triangulate(poly[k:] + poly[:1]) if k < n - 1 else []
        if left is not None and right is not None:
            return [(poly[0], poly[1], poly[k])] + left + right
    return None


def case_triangles(case):
    nxt = {}
    for e0, e1 in segments(case):
        assert e0 not in nxt, (case, e0)
        nxt[e0] = e1
    assert sorted(nxt) == sorted(nxt.values()), case
    tris = []
    for start in sorted(nxt):
        if start not in nxt:
            continue
        loop, e = [], start
        while e in nxt:
            loop.append(e)
            e = nxt.pop(e)
        t = triangulate(loop)
        assert t is not None, (case, loop)
        tris += t
    return tris


def table():
    return [case_triangles(c) for c in range(256)]


def main():
    tab = table()
    max_tris = max(len(t) for t in tab)
    assert max_tris <= MAX_TRIS, max_tris
    row = 3 * MAX_TRIS
    lines = ["// Generated by mcubes_table.py from its face rule; do not edit.  The rows of an initialiser (mcubes.cu includes",
             "// this file inside the braces of its table definitions): row c = the triangles of case c as edge ids, three",
             "// per triangle, padded with -1 to %d entries." % row]
    for c, tris in enumerate(tab):
        flat = [e for t in tris for e in t] + [-1] * (row - 3 * len(tris))
        lines.append("    {%s},  // %d" % (", ".join(str(v) for v in flat), c))
    out = os.path.join(os.path.dirname(os.path.abspath(__file__)), "mcubes_table.cuh")
    with open(out, "w") as f:
        f.write("\n".join(lines) + "\n")
    print("%s: max %d triangles per case" % (out, max_tris))


if __name__ == "__main__":
    main()
