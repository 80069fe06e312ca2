"""Exact-rational referee of the clip of line and point rows by polygon rows (DESIGN.md §4.22) — TEST INFRASTRUCTURE ONLY.

Reached by another route than the kernel, in fractions.Fraction:
  1. every line segment is cut at the parameter of every meeting with every polygon edge (crossings and the ends of collinear
     overlaps, relate_reference._meet_params);
  2. every sub-piece is classified by its midpoint with the exact in / on / out test relate_reference.locate;
  3. the kept pieces of one chain are merged into runs by the output rules: intersection keeps a run through a point where the
     line touches the boundary, difference splits it there; runs never cross chains.
A member is a list of (point, tol): an input vertex (of the line or the polygon) has tol 0 and must match bit for bit, a
crossing has the rounding bound of the kernel's a0 + t (a1 - a0).  Pure-Python loops: small cases only.  Valid polygons only.
"""
from __future__ import annotations

import math
from fractions import Fraction as F

import relate_reference as rr

EPS = 2.0**-53


def _chains(kind, row):
    mem = [row] if kind == "linestring" else list(row)
    return [[(F(p[0]), F(p[1])) for p in ch] for ch in mem]


def _ulp(x):
    return math.ulp(abs(x)) if x else 5e-324


def _tol(e, f, cmax, L):
    """rounding bound of the crossing of the line segment e with the polygon edge f"""
    le = math.hypot(float(e[1][0] - e[0][0]), float(e[1][1] - e[0][1]))
    lf = math.hypot(float(f[1][0] - f[0][0]), float(f[1][1] - f[0][1]))
    cr = abs(rr._cross(e[1][0] - e[0][0], e[1][1] - e[0][1], f[1][0] - f[0][0], f[1][1] - f[0][1]))
    return 2 * _ulp(cmax) + 16 * EPS * L * le * lf / float(cr) if cr else 2 * _ulp(cmax)


def clip(kind_a, a_row, kind_b, b_row, invert=False):
    """the members of clip(a, b): for lines a list of members, each a list of (point, tol); for points a list of points"""
    gb = rr.parse(kind_b, b_row)
    if kind_a in ("point", "multipoint"):
        pts = [a_row] if kind_a == "point" else list(a_row)
        keep = [(rr.locate(gb, (F(p[0]), F(p[1]))) == rr.E) == invert for p in pts]
        return [p for p, k in zip(pts, keep) if k]
    segs = rr._segments(gb)
    verts = set(rr._vertices(gb))
    chains = _chains(kind_a, a_row)
    coords = [abs(float(c)) for ch in chains for p in ch for c in p] + [abs(float(c)) for p in verts for c in p] + [1.0]
    cmax = max(coords)
    xs = [float(p[0]) for ch in chains for p in ch] + [float(p[0]) for p in verts]
    ys = [float(p[1]) for ch in chains for p in ch] + [float(p[1]) for p in verts]
    L = math.hypot(max(xs) - min(xs), max(ys) - min(ys)) if xs else 0.0
    out = []
    for ch in chains:
        lverts = set(ch)
        run, prev_kept = [], False
        for i in range(len(ch) - 1):
            p0, p1 = ch[i], ch[i + 1]
            if p0 == p1:
                continue
            cuts = {F(0): None, F(1): None}
            for s in segs:
                for t in rr._meet_params(p0, p1, s[0], s[1]):
                    if t not in cuts or cuts[t] is None:
                        cuts[t] = s
            ts = sorted(cuts)
            pt = lambda t: (p0[0] + t * (p1[0] - p0[0]), p0[1] + t * (p1[1] - p0[1]))  # noqa: E731

            def tagged(t):
                q = pt(t)
                if q in lverts or q in verts:
                    return (q, 0.0)
                return (q, _tol((p0, p1), cuts[t], cmax, L))

            for t0, t1 in zip(ts, ts[1:]):
                mid = pt((t0 + t1) / 2)
                loc = rr.locate(gb, mid)
                kept = (loc == rr.E) == invert
                start_on = rr.locate(gb, pt(t0)) != rr.E
                if kept and prev_kept and not (invert and start_on):
                    run.append(tagged(t1))
                else:
                    if len(run) >= 2:
                        out.append(run)
                    run = [tagged(t0), tagged(t1)] if kept else []
                prev_kept = kept
        if len(run) >= 2:
            out.append(run)
    return out


def length(kind_a, a_row, kind_b, b_row, invert=False):
    """the exact length of the clip, as a sum of float lengths of its exact pieces (Fractions squared, then one sqrt each)"""
    tot = 0.0
    for m in clip(kind_a, a_row, kind_b, b_row, invert):
        for (p, _), (q, _) in zip(m, m[1:]):
            tot += math.sqrt(float((q[0] - p[0]) ** 2 + (q[1] - p[1]) ** 2))
    return tot


def matches(got, want):
    """a kernel member list (lists of (x, y) floats) against the referee's: same members, same vertex counts, input vertices
    bit for bit and cut points within their bound.  Returns None, or a message"""
    if len(got) != len(want):
        return "%d members, referee %d" % (len(got), len(want))
    for k, (g, w) in enumerate(zip(got, want)):
        if len(g) != len(w):
            return "member %d: %d points, referee %d" % (k, len(g), len(w))
        for (gx, gy), (p, tol) in zip(g, w):
            wx, wy = float(p[0]), float(p[1])
            if tol == 0.0:
                if (gx, gy) != (wx, wy):
                    return "member %d: vertex (%r, %r) != (%r, %r)" % (k, gx, gy, wx, wy)
            elif abs(gx - wx) > tol or abs(gy - wy) > tol:
                return "member %d: cut point (%r, %r) beyond %g of (%r, %r)" % (k, gx, gy, tol, wx, wy)
    return None


# ---- hand cases: (name, kind_a, a, kind_b, b, intersection members, difference members), exact ------------------------------
SQ = [(0.0, 0.0), (4.0, 0.0), (4.0, 4.0), (0.0, 4.0), (0.0, 0.0)]
ELL = [(0.0, 0.0), (4.0, 0.0), (4.0, 2.0), (2.0, 2.0), (2.0, 4.0), (0.0, 4.0), (0.0, 0.0)]  # reflex vertex at (2, 2)
HOLED = [[(0.0, 0.0), (8.0, 0.0), (8.0, 8.0), (0.0, 8.0), (0.0, 0.0)], [(2.0, 2.0), (2.0, 6.0), (6.0, 6.0), (6.0, 2.0), (2.0, 2.0)]]
HAND = [
    ("through_square", "linestring", [(-2.0, 2.0), (6.0, 2.0)], "polygon", [SQ],
     [[(0.0, 2.0), (4.0, 2.0)]], [[(-2.0, 2.0), (0.0, 2.0)], [(4.0, 2.0), (6.0, 2.0)]]),
    ("along_edge", "linestring", [(1.0, 0.0), (3.0, 0.0)], "polygon", [SQ], [[(1.0, 0.0), (3.0, 0.0)]], []),
    ("along_edge_beyond", "linestring", [(-1.0, 0.0), (5.0, 0.0)], "polygon", [SQ],
     [[(0.0, 0.0), (4.0, 0.0)]], [[(-1.0, 0.0), (0.0, 0.0)], [(4.0, 0.0), (5.0, 0.0)]]),
    ("touch_vertex", "linestring", [(3.0, 5.0), (5.0, 3.0)], "polygon", [SQ], [], [[(3.0, 5.0), (4.0, 4.0)], [(4.0, 4.0), (5.0, 3.0)]]),
    ("reflex_vertex", "linestring", [(1.0, 3.0), (3.0, 1.0)], "polygon", [ELL], [[(1.0, 3.0), (2.0, 2.0), (3.0, 1.0)]], []),
    ("across_hole", "linestring", [(-1.0, 4.0), (9.0, 4.0)], "polygon", HOLED,
     [[(0.0, 4.0), (2.0, 4.0)], [(6.0, 4.0), (8.0, 4.0)]], [[(-1.0, 4.0), (0.0, 4.0)], [(2.0, 4.0), (6.0, 4.0)], [(8.0, 4.0), (9.0, 4.0)]]),
    ("closed_inside", "linestring", [(1.0, 1.0), (3.0, 1.0), (3.0, 3.0), (1.0, 3.0), (1.0, 1.0)], "polygon", [SQ],
     [[(1.0, 1.0), (3.0, 1.0), (3.0, 3.0), (1.0, 3.0), (1.0, 1.0)]], []),
    ("closed_crossing", "linestring", [(1.0, 1.0), (6.0, 1.0), (6.0, 3.0), (1.0, 3.0), (1.0, 1.0)], "polygon", [SQ],
     [[(1.0, 1.0), (4.0, 1.0)], [(4.0, 3.0), (1.0, 3.0), (1.0, 1.0)]], [[(4.0, 1.0), (6.0, 1.0), (6.0, 3.0), (4.0, 3.0)]]),
    ("starts_on_boundary", "linestring", [(0.0, 2.0), (2.0, 2.0), (2.0, 6.0)], "polygon", [SQ],
     [[(0.0, 2.0), (2.0, 2.0), (2.0, 4.0)]], [[(2.0, 4.0), (2.0, 6.0)]]),
    ("zero_length_segments", "linestring", [(-2.0, 2.0), (-2.0, 2.0), (1.0, 2.0), (1.0, 2.0), (6.0, 2.0)], "polygon", [SQ],
     [[(0.0, 2.0), (1.0, 2.0), (4.0, 2.0)]], [[(-2.0, 2.0), (0.0, 2.0)], [(4.0, 2.0), (6.0, 2.0)]]),
    ("multi_both_sides", "multilinestring", [[(-2.0, 1.0), (-1.0, 1.0)], [(1.0, 1.0), (3.0, 3.0)], [(5.0, 5.0), (6.0, 6.0)]], "polygon", [SQ],
     [[(1.0, 1.0), (3.0, 3.0)]], [[(-2.0, 1.0), (-1.0, 1.0)], [(5.0, 5.0), (6.0, 6.0)]]),
    ("points", "multipoint", [(2.0, 2.0), (4.0, 1.0), (5.0, 5.0), (0.0, 0.0), (2.0, 2.0)], "polygon", [SQ],
     [(2.0, 2.0), (4.0, 1.0), (0.0, 0.0), (2.0, 2.0)], [(5.0, 5.0)]),
]


def plain(members):
    """the referee's line members as lists of float points"""
    return [[(float(p[0]), float(p[1])) for p, _ in m] for m in members]


def l1(members):
    """the exact L1 length of line members (additive along a segment, so the exact partition identity holds in it)"""
    return sum((abs(q[0] - p[0]) + abs(q[1] - p[1]) for m in members for (p, _), (q, _) in zip(m, m[1:])), F(0))
