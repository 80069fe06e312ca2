"""Exact-rational referee for the intersection area of two (Multi)Polygons — TEST INFRASTRUCTURE ONLY.

Cut and classify on the exact arrangement, a formulation deliberately different from the kernel's (DESIGN.md §4.16):
every boundary edge is cut at its meetings with the other side's boundary (oracle.exact._cut_params); a piece of
boundary(A) counts when its midpoint is strictly inside B, or lies on boundary(B) running in the same direction (both
interiors on the same side); a piece of boundary(B) counts when its midpoint is strictly inside A.  The counted pieces,
each oriented with its own region's interior on the left, are the boundary of A ∩ B, and half the sum of their cross
products is its area.  Ring orientation comes from the exact shoelace sum (the kernel uses the turn at the lowest vertex).
Every value is a fractions.Fraction; pure-Python loops, small cases only.  Valid (OGC) operands only.
"""
from __future__ import annotations

from fractions import Fraction as F

from oracle import exact


def _shoelace2(ring):
    return sum(F(s[0]) * F(e[1]) - F(e[0]) * F(s[1]) for s, e in zip(ring[:-1], ring[1:]))


def _usable(members):
    """members with their rings closed; rings with fewer than 4 coordinates after closing are dropped (a member whose
    exterior is dropped goes with it)"""
    out = []
    for rings in members:
        rr = [exact._closed(r) for r in rings]
        if not rr or len(rr[0]) < 4:
            continue
        out.append([r for r in rr if len(r) >= 4])
    return out


def _oriented_edges(members):
    """every non-degenerate boundary edge, oriented with the region's interior on its left"""
    edges = []
    for rings in members:
        for k, r in enumerate(rings):
            a2 = _shoelace2(r)
            if a2 == 0:
                continue
            ccw = a2 > 0
            forward = ccw if k == 0 else not ccw
            for s, e in zip(r[:-1], r[1:]):
                if tuple(s) != tuple(e):
                    edges.append((tuple(s), tuple(e)) if forward else (tuple(e), tuple(s)))
    return edges


def _pieces(u, v, others):
    ts = exact._cut_params(u, v, others)
    ux, uy, vx, vy = map(F, (*u, *v))
    for t0, t1 in zip(ts[:-1], ts[1:]):
        a = (ux + t0 * (vx - ux), uy + t0 * (vy - uy))
        b = (ux + t1 * (vx - ux), uy + t1 * (vy - uy))
        m = ((a[0] + b[0]) / 2, (a[1] + b[1]) / 2)
        yield a, b, m


def _same_direction_on(m, u, v, edges):
    """m lies on an edge of `edges` that runs in the direction of u -> v"""
    dx, dy = F(v[0]) - F(u[0]), F(v[1]) - F(u[1])
    for s, e in edges:
        if exact._on_segment(m, s, e):
            ex, ey = F(e[0]) - F(s[0]), F(e[1]) - F(s[1])
            if ex * dy - ey * dx == 0 and ex * dx + ey * dy > 0:
                return True
    return False


def intersection_area(a_members, b_members) -> F:
    """area of closed(A) ∩ closed(B); A, B: lists of polygons, each a list of rings (closed or not, any orientation)"""
    am, bm = _usable(a_members), _usable(b_members)
    ea, eb = _oriented_edges(am), _oriented_edges(bm)
    if not ea or not eb:
        return F(0)
    total = F(0)
    for u, v in ea:
        for a, b, m in _pieces(u, v, eb):
            pos = exact._region_pos(m, bm)
            if pos == 2 or (pos == 1 and _same_direction_on(m, u, v, eb)):
                total += a[0] * b[1] - b[0] * a[1]
    for u, v in eb:
        for a, b, m in _pieces(u, v, ea):
            if exact._region_pos(m, am) == 2:
                total += a[0] * b[1] - b[0] * a[1]
    return total / 2


def polygon_area(members) -> F:
    """exact area of a valid (Multi)Polygon: exteriors minus holes"""
    tot = F(0)
    for rings in _usable(members):
        for k, r in enumerate(rings):
            a = abs(_shoelace2(r)) / 2
            tot += a if k == 0 else -a
    return tot
