"""Exact-rational referee of the DE-9IM matrix (DESIGN.md §4.20) — TEST INFRASTRUCTURE ONLY.

Built by a route other than the kernel's, on the noded arrangement in fractions.Fraction:
  1. every segment of both operands (rings closed as Polygon::new closes them) is cut at its rational meetings with every
     other segment, of either operand: crossing points and the ends of collinear overlaps;
  2. samples: every vertex, cut point and point member (dimension 0), the midpoint of every sub-segment (dimension 1) and
     both side-offsets of every midpoint (dimension 2), the offset halved until the segment from the midpoint to it meets
     no segment except at the midpoint;
  3. every sample is located exactly in both operands (I / B / E; a line's boundary by the Mod-2 rule, a polygon's is its
     rings) and each (locA, locB) cell keeps the largest sample dimension.  EE is always 2.
Pure-Python loops: small cases only.  Valid (OGC) operands only.
"""
from __future__ import annotations

from fractions import Fraction as F

I, B, E = 0, 1, 2
CLASS = {"point": 0, "multipoint": 0, "linestring": 1, "multilinestring": 1, "polygon": 2, "multipolygon": 2}


def parse(kind, row):
    """(class, points, chains, polygons) with Fraction coordinates; chains / rings as lists of points, rings closed"""
    c = CLASS[kind]
    mem = [row] if kind in ("point", "linestring", "polygon") else list(row)
    fr = lambda p: (F(p[0]), F(p[1]))  # noqa: E731
    pts, chains, polys = [], [], []
    if c == 0:
        pts = [fr(p) for p in mem]
    elif c == 1:
        chains = [[fr(p) for p in m] for m in mem]
    else:
        for poly in mem:
            rings = []
            for r in poly:
                q = [fr(p) for p in r]
                if q and q[0] != q[-1]:
                    q.append(q[0])
                rings.append(q)
            polys.append(rings)
    return c, pts, chains, polys


def _segments(g):
    c, pts, chains, polys = g
    out = []
    for ch in chains:
        out += [(ch[i], ch[i + 1]) for i in range(len(ch) - 1)]
    for rings in polys:
        for r in rings:
            out += [(r[i], r[i + 1]) for i in range(len(r) - 1)]
    return [s for s in out if s[0] != s[1]]


def _vertices(g):
    c, pts, chains, polys = g
    out = list(pts)
    for ch in chains:
        out += ch
    for rings in polys:
        for r in rings:
            out += r
    return out


def _cross(ax, ay, bx, by):
    return ax * by - ay * bx


def _orient(a, b, p):
    return _cross(b[0] - a[0], b[1] - a[1], p[0] - a[0], p[1] - a[1])


def _on_segment(p, s, e):
    return _orient(s, e, p) == 0 and min(s[0], e[0]) <= p[0] <= max(s[0], e[0]) and min(s[1], e[1]) <= p[1] <= max(s[1], e[1])


def _meet_params(p0, p1, q0, q1):
    """parameters t on p0-p1 of the points where the closed segments p0-p1 and q0-q1 meet (crossing or overlap ends)"""
    dx, dy = p1[0] - p0[0], p1[1] - p0[1]
    ex, ey = q1[0] - q0[0], q1[1] - q0[1]
    d = _cross(dx, dy, ex, ey)
    wx, wy = q0[0] - p0[0], q0[1] - p0[1]
    if d != 0:
        t, u = _cross(wx, wy, ex, ey) / d, _cross(wx, wy, dx, dy) / d
        return [t] if 0 <= t <= 1 and 0 <= u <= 1 else []
    if _cross(wx, wy, dx, dy) != 0:
        return []
    ll = dx * dx + dy * dy
    ts = [((q[0] - p0[0]) * dx + (q[1] - p0[1]) * dy) / ll for q in (q0, q1)]
    out = [t for t in ts if 0 <= t <= 1]
    if _on_segment(p0, q0, q1):
        out.append(F(0))
    if _on_segment(p1, q0, q1):
        out.append(F(1))
    return out


def _ring_inside(p, ring):
    """even-odd crossing test of a point not on the ring"""
    inside = False
    for i in range(len(ring) - 1):
        a, b = ring[i], ring[i + 1]
        if (a[1] > p[1]) != (b[1] > p[1]):
            x = a[0] + (p[1] - a[1]) * (b[0] - a[0]) / (b[1] - a[1])
            if x > p[0]:
                inside = not inside
    return inside


def locate(g, p):
    c, pts, chains, polys = g
    if c == 0:
        return I if p in pts else E
    if c == 1:
        if not any(_on_segment(p, ch[i], ch[i + 1]) for ch in chains for i in range(len(ch) - 1)):
            return E
        ends = sum((ch[0] == p) + (ch[-1] == p) for ch in chains if len(ch) >= 2)
        return B if ends % 2 else I
    for rings in polys:
        for r in rings:
            if any(_on_segment(p, r[i], r[i + 1]) for i in range(len(r) - 1)):
                return B
    for rings in polys:
        if rings and len(rings[0]) >= 4 and _ring_inside(p, rings[0]) and not any(_ring_inside(p, h) for h in rings[1:]):
            return I
    return E


def _clear(m, q, segs):
    """the closed segment m-q meets no segment except at m"""
    for s, e in segs:
        for t in _meet_params(m, q, s, e):
            if t != 0:
                return False
    return True


def relate(kind_a, a_row, kind_b, b_row) -> str:
    """the DE-9IM matrix as a 9-character string over F012"""
    A, Bg = parse(kind_a, a_row), parse(kind_b, b_row)
    M = [[-1] * 3 for _ in range(3)]
    M[E][E] = 2

    def add(p, d):
        la, lb = locate(A, p), locate(Bg, p)
        M[la][lb] = max(M[la][lb], d)

    segs = _segments(A) + _segments(Bg)
    # point members cut the segments they lie on and must stay off the offset paths: degenerate segments
    others = segs + [(p, p) for g in (A, Bg) for p in g[1]]
    for p in _vertices(A) + _vertices(Bg):
        add(p, 0)
    for i, (p0, p1) in enumerate(segs):
        ts = {F(0), F(1)}
        for j, (q0, q1) in enumerate(others):
            if i != j:
                ts.update(_meet_params(p0, p1, q0, q1))
        ts = sorted(ts)
        dx, dy = p1[0] - p0[0], p1[1] - p0[1]
        for t in ts:
            add((p0[0] + t * dx, p0[1] + t * dy), 0)
        for t0, t1 in zip(ts, ts[1:]):
            tm = (t0 + t1) / 2
            m = (p0[0] + tm * dx, p0[1] + tm * dy)
            add(m, 1)
            for sgn in (1, -1):
                h = F(1, 2)
                while True:
                    q = (m[0] - sgn * h * dy, m[1] + sgn * h * dx)
                    if _clear(m, q, others):
                        break
                    h /= 2
                add(q, 2)
    return "".join("F" if v < 0 else str(v) for row in M for v in row)


def matches(matrix: str, pattern: str) -> bool:
    for m, p in zip(matrix, pattern.upper()):
        if p == "*":
            continue
        if p == "T" and m == "F":
            return False
        if p in "F012" and m != p:
            return False
    return True


def dims(kind):
    return CLASS[kind]


def predicate(name, matrix, da, db, empty_a=False, empty_b=False, pattern=None) -> bool:
    """JTS's named predicates on a matrix (dims: the operands' type dimensions)"""
    any_of = lambda *ps: any(matches(matrix, p) for p in ps)  # noqa: E731
    if name == "intersects":
        return not matches(matrix, "FF*FF****")
    if name == "disjoint":
        return matches(matrix, "FF*FF****")
    if name == "contains":
        return any_of("T*****FF*")
    if name == "within":
        return any_of("T*F**F***")
    if name == "contains_properly":
        return any_of("T**FF*FF*")
    if name == "covers":
        return any_of("T*****FF*", "*T****FF*", "***T**FF*", "****T*FF*")
    if name == "covered_by":
        return any_of("T*F**F***", "*TF**F***", "**FT*F***", "**F*TF***")
    if name == "touches":
        return not (da == 0 and db == 0) and any_of("FT*******", "F**T*****", "F***T****")
    if name == "crosses":
        if da < db:
            return any_of("T*T******")
        if da > db:
            return any_of("T*****T**")
        return da == 1 and any_of("0********")
    if name == "overlaps":
        if da != db:
            return False
        return any_of("1*T***T**" if da == 1 else "T*T***T**")
    if name == "geom_equals":
        if empty_a and empty_b:
            return True
        return da == db and any_of("T*F**FFF*")
    if name == "relate_pattern":
        return matches(matrix, pattern)
    raise ValueError(name)


def transpose(m: str) -> str:
    return "".join(m[3 * c + r] for r in range(3) for c in range(3))
