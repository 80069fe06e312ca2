"""Exact-rational referee of the OGC validity codes of gpl_is_valid (DESIGN.md §4.18) — TEST INFRASTRUCTURE ONLY.

It follows the contract by routes other than the kernel's:
  - edge pairs: parametric intersection of the two segments in Fractions (t, u of both lines), after a numpy box sweep and a
    floating-point filter that only drops pairs it can certify disjoint (or adjacent edges certified to meet only at their
    shared vertex);
  - ring in ring: even-odd ray casting of an exact rational point, the midpoint of the first piece of the ring's first edge
    (from its start to the nearest point of the edge where another ring touches it);
  - disconnected interior: face counting of the planar arrangement of one polygon's rings, split at their touch points.
    With V vertices, E edges and C components the bounded faces number E - V + C; the interior is connected iff that equals
    the number of rings.
Rows are given in the nesting GeoArrowArray.from_shapes takes; None is a null row (code None).
"""
from __future__ import annotations

import math
import os
import sys
from fractions import Fraction as F

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from oracle.exact import orient_sign  # noqa: E402

MESSAGES = {0: "Valid Geometry", 2: "Hole lies outside shell", 3: "Holes are nested", 4: "Interior is disconnected", 5: "Self-intersection",
            6: "Ring Self-intersection", 7: "Nested shells", 9: "Too few distinct points in geometry component", 10: "Invalid Coordinate"}


def _fin(p):
    return math.isfinite(p[0]) and math.isfinite(p[1])


def ring_vertices(ring):
    """the distinct consecutive vertices of a ring, closed implicitly (cyclic, first vertex first)"""
    pts = [tuple(map(float, p)) for p in ring]
    if not pts:
        return []
    if pts[0] != pts[-1]:
        pts.append(pts[0])
    out = [pts[0]]
    for p in pts[1:]:
        if p != out[-1]:
            out.append(p)
    if len(out) > 1 and out[-1] == out[0]:
        out.pop()
    return out


def _cross(ax, ay, bx, by):
    return ax * by - ay * bx


def segment_relation(p, q, r, s):
    """exact: (0, None) disjoint, (1, None) proper crossing or overlap of positive length, (2, X) one common point X"""
    px, py, qx, qy, rx, ry, sx, sy = map(F, (*p, *q, *r, *s))
    dx, dy, ex, ey = qx - px, qy - py, sx - rx, sy - ry
    den = _cross(dx, dy, ex, ey)
    wx, wy = rx - px, ry - py
    if den != 0:
        t = _cross(wx, wy, ex, ey) / den
        u = _cross(wx, wy, dx, dy) / den
        if not (0 <= t <= 1 and 0 <= u <= 1):
            return 0, None
        if 0 < t < 1 and 0 < u < 1:
            return 1, None
        return 2, (px + t * dx, py + t * dy)
    if _cross(wx, wy, dx, dy) != 0:
        return 0, None
    dd = dx * dx + dy * dy
    t0 = (wx * dx + wy * dy) / dd
    t1 = ((sx - px) * dx + (sy - py) * dy) / dd
    lo, hi = max(F(0), min(t0, t1)), min(F(1), max(t0, t1))
    if lo < hi:
        return 1, None
    if lo > hi:
        return 0, None
    return 2, (px + lo * dx, py + lo * dy)


def _certain_signs(ax, ay, bx, by, cx, cy):
    """numpy orient2d signs with a stage-A error bound: (sign, certain)"""
    dl = (ax - cx) * (by - cy)
    dr = (ay - cy) * (bx - cx)
    det = dl - dr
    ok = np.abs(det) > 3.3306690738754716e-16 * (np.abs(dl) + np.abs(dr))
    return np.sign(det) * ok, ok


def _candidate_pairs(E):
    """index pairs i < j of edges (array n x 4: x0 y0 x1 y1) whose closed boxes meet: sweep on x, numpy"""
    n = len(E)
    if n < 2:
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    bx0, bx1 = np.minimum(E[:, 0], E[:, 2]), np.maximum(E[:, 0], E[:, 2])
    by0, by1 = np.minimum(E[:, 1], E[:, 3]), np.maximum(E[:, 1], E[:, 3])
    order = np.argsort(bx0, kind="stable")
    sx0 = bx0[order]
    hi = np.searchsorted(sx0, bx1[order], side="right")
    pos = np.arange(n)
    cnt = np.maximum(hi - pos - 1, 0)
    a = np.repeat(pos, cnt)
    start = np.repeat(pos + 1 - np.concatenate([[0], np.cumsum(cnt)[:-1]]), cnt)
    b = np.arange(len(a)) + start
    ia, ib = order[a], order[b]
    keep = (by0[ia] <= by1[ib]) & (by0[ib] <= by1[ia])
    ia, ib = ia[keep], ib[keep]
    return np.minimum(ia, ib), np.maximum(ia, ib)


def _inside_even_odd(m, ring):
    """exact even-odd test of the rational point m against a ring of distinct consecutive vertices; m on the ring: error"""
    mx, my = m
    n = len(ring)
    A = np.array(ring, float)
    B = np.roll(A, -1, axis=0)
    fy = float(my)
    sel = np.nonzero((np.minimum(A[:, 1], B[:, 1]) <= fy + 1e-9 * (1 + abs(fy))) & (np.maximum(A[:, 1], B[:, 1]) >= fy - 1e-9 * (1 + abs(fy))))[0]
    inside = False
    for i in sel:
        (ax, ay), (bx, by) = ring[i], ring[(i + 1) % n]
        ax, ay, bx, by = F(ax), F(ay), F(bx), F(by)
        if (ay > my) != (by > my):
            x = ax + (my - ay) * (bx - ax) / (by - ay)
            assert x != mx, "test point on a ring"
            if x > mx:
                inside = not inside
        elif ay == my == by:
            assert not (min(ax, bx) <= mx <= max(ax, bx)), "test point on a ring"
    return inside


def _box(ring):
    a = np.array(ring, float)
    return a[:, 0].min(), a[:, 1].min(), a[:, 0].max(), a[:, 1].max()


def _in_box(m, b):
    return b[0] <= float(m[0]) <= b[2] and b[1] <= float(m[1]) <= b[3]


def polygon_code(polys):
    """rules 9, 5, 6, 2, 3, 7, 4 of a list of polygons (each a list of rings), coordinates finite"""
    rings = []  # (poly, ring index in poly, vertices)
    for pi, poly in enumerate(polys):
        for ri, ring in enumerate(poly):
            if len(ring) == 0:
                rings.append((pi, ri, []))
                continue
            v = ring_vertices(ring)
            if len(v) < 3:
                return 9
            rings.append((pi, ri, v))
    edges, meta = [], []  # meta: (ring id, index in ring)
    for g, (_, _, v) in enumerate(rings):
        for i in range(len(v)):
            edges.append((*v[i], *v[(i + 1) % len(v)]))
            meta.append((g, i))
    E = np.array(edges, float).reshape(-1, 4)
    meta = np.array(meta, np.int64).reshape(-1, 2)
    ia, ib = _candidate_pairs(E)
    # floating-point filter: drop pairs certified disjoint, and adjacent edges of a ring certified to meet only at their vertex
    p, q, r, s = E[ia, 0:2], E[ia, 2:4], E[ib, 0:2], E[ib, 2:4]
    o1, c1 = _certain_signs(p[:, 0], p[:, 1], q[:, 0], q[:, 1], r[:, 0], r[:, 1])
    o2, c2 = _certain_signs(p[:, 0], p[:, 1], q[:, 0], q[:, 1], s[:, 0], s[:, 1])
    o3, c3 = _certain_signs(r[:, 0], r[:, 1], s[:, 0], s[:, 1], p[:, 0], p[:, 1])
    o4, c4 = _certain_signs(r[:, 0], r[:, 1], s[:, 0], s[:, 1], q[:, 0], q[:, 1])
    drop = (c1 & c2 & (o1 * o2 > 0)) | (c3 & c4 & (o3 * o4 > 0))
    ga, gb = meta[ia, 0], meta[ib, 0]
    k = np.array([len(rings[g][2]) for g in range(len(rings))], np.int64)
    same = ga == gb
    d = (meta[ib, 1] - meta[ia, 1]) % np.maximum(k[ga], 1)
    nxt = same & (d == 1)  # edge b starts where edge a ends: shared vertex q == r; they meet only there unless p, q, s collinear
    prv = same & (d == k[ga] - 1)  # edge a starts where b ends: p == s
    drop |= nxt & c2 & (o2 != 0)
    drop |= prv & c1 & (o1 != 0)
    ia, ib = ia[~drop], ib[~drop]
    flags = set()
    touches = {}  # poly -> list of (ring a, ring b, point)
    splits = {}  # edge -> set of points strictly inside it
    for a, b in zip(ia.tolist(), ib.tolist()):
        rel, X = segment_relation(E[a, 0:2], E[a, 2:4], E[b, 0:2], E[b, 2:4])
        if rel == 0:
            continue
        if rel == 1:
            return 5
        (g1, i1), (g2, i2) = meta[a], meta[b]
        if g1 == g2:
            kk = len(rings[g1][2])
            if (i2 - i1) % kk not in (1, kk - 1):
                flags.add(6)
        elif rings[g1][0] == rings[g2][0]:
            touches.setdefault(rings[g1][0], []).append((int(g1), int(g2), X))
            for e in (a, b):
                ends = {(F(E[e, 0]), F(E[e, 1])), (F(E[e, 2]), F(E[e, 3]))}
                if X not in ends:
                    splits.setdefault(e, set()).add(X)
    if 6 in flags:
        return 6
    # ring in ring
    by_poly = {}
    for g, (pi, ri, v) in enumerate(rings):
        by_poly.setdefault(pi, []).append(g)
    boxes = [(_box(v) if v else None) for (_, _, v) in rings]

    def test_point(g):
        v = rings[g][2]
        (ux, uy), (wx, wy) = v[0], v[1]
        ux, uy, wx, wy = F(ux), F(uy), F(wx), F(wy)
        dx, dy = wx - ux, wy - uy
        dd = dx * dx + dy * dy
        tmin = F(1)
        for h, (_, _, vh) in enumerate(rings):
            if h == g or not vh or not (boxes[h][0] <= max(v[0][0], v[1][0]) and min(v[0][0], v[1][0]) <= boxes[h][2]
                                       and boxes[h][1] <= max(v[0][1], v[1][1]) and min(v[0][1], v[1][1]) <= boxes[h][3]):
                continue
            for c in vh:
                cx, cy = F(c[0]), F(c[1])
                if _cross(cx - ux, cy - uy, dx, dy) == 0:
                    t = ((cx - ux) * dx + (cy - uy) * dy) / dd
                    if 0 < t < tmin:
                        tmin = t
        return (ux + tmin / 2 * dx, uy + tmin / 2 * dy)
    for pi, lst in by_poly.items():
        shell = lst[0]
        for h in lst[1:]:
            if not rings[h][2]:
                continue
            m = test_point(h)
            if not rings[shell][2] or not (_in_box(m, boxes[shell]) and _inside_even_odd(m, rings[shell][2])):
                flags.add(2)
            for o in lst[1:]:
                if o != h and rings[o][2] and _in_box(m, boxes[o]) and _inside_even_odd(m, rings[o][2]):
                    flags.add(3)
    if len(polys) > 1:
        for pi, lst in by_poly.items():
            if not rings[lst[0]][2]:
                continue
            m = test_point(lst[0])
            for pj, lj in by_poly.items():
                if pj == pi or not rings[lj[0]][2]:
                    continue
                if _in_box(m, boxes[lj[0]]) and _inside_even_odd(m, rings[lj[0]][2]):
                    if not any(rings[h][2] and _in_box(m, boxes[h]) and _inside_even_odd(m, rings[h][2]) for h in lj[1:]):
                        flags.add(7)
    for c in (2, 3, 7):
        if c in flags:
            return c
    # disconnected interior: face counting per polygon
    for pi, lst in touches.items():
        rl = [g for g in by_poly[pi] if rings[g][2]]
        verts = set()
        n_edges = 0
        for g in rl:
            verts.update((F(x), F(y)) for x, y in rings[g][2])
        for e in range(len(E)):
            if meta[e, 0] in rl:
                n_edges += 1 + len(splits.get(e, ()))
        parent = {g: g for g in rl}  # components of the ring graph (rings joined by a touch)
        def find(x):
            while parent[x] != x:
                x = parent[x]
            return x
        for a, b, _ in lst:
            parent[find(a)] = find(b)
        comps = len({find(g) for g in rl})
        if n_edges - len(verts) + comps != len(rl):
            return 4
    return 0


def validity_code(kind, geom):
    """the reason code of one row (kind: point, multipoint, linestring, multilinestring, polygon, multipolygon)"""
    if geom is None:
        return None
    if kind == "point":
        x, y = map(float, geom)
        if math.isnan(x) and math.isnan(y):
            return 0
        return 0 if _fin((x, y)) else 10
    if kind == "multipoint":
        return 0 if all(_fin(p) for p in geom) else 10
    if kind in ("linestring", "multilinestring"):
        lines = [geom] if kind == "linestring" else geom
        if not all(_fin(p) for ln in lines for p in ln):
            return 10
        return 9 if any(len(ln) > 0 and len({tuple(p) for p in ln}) < 2 for ln in lines) else 0
    polys = [geom] if kind == "polygon" else geom
    if not all(_fin(p) for poly in polys for ring in poly for p in ring):
        return 10
    return polygon_code(polys)
