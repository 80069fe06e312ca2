"""Exact referee for the row-wise pair operations `intersects`, `distance` and `contains` — TEST INFRASTRUCTURE ONLY.

It works on the exact values of the input doubles.  Every finite double is a dyadic rational, so the coordinates of one row
pair are scaled by a common power of two to Python integers, and every decision and every squared distance is then an exact
integer or rational computation.  The polygon predicates are those of oracle/exact.py (ray casting and exact arrangements),
called on the scaled integers; the chain predicates are exact orientation signs.  Scope: VALID geometry only (OGC-valid
polygons, linestrings of >= 2 coordinates); null, empty, 1-coordinate and invalid rows are not defined here.

Rows are in the nesting `GeoArrowArray.from_shapes` takes; `kind` is one of tests/shapes.KINDS.

Semantics (DESIGN §4.5, §4.10):
* `intersects`: the closed point sets share a point; a Multi* row is the union of its members.
* `distance2`: the exact squared Euclidean distance of the closed point sets: 0 when they intersect, else the minimum over
  (vertex, segment) pairs in both directions over every ring (holes included) and every member — for disjoint closed sets
  bounded by segments the minimum is reached at a vertex of one of them.
* `contains_point`: (Multi)Polygon: the point is in the interior of a member; (Multi)LineString: the point is on a member and
  is not an end point of an open member (geo's `Contains<Coord>`).
* `contains_polygon`: (Multi)Polygon contains Polygon, DE-9IM [T*****FF*].

The distance error bound.  The kernels evaluate, per (vertex p, segment s-e) pair with 0 < r < 1,
    cross = (s.y - p.y)·dx - (s.x - p.x)·dy,   d² = cross² / (dx² + dy²),
and the vertex cases as dx² + dy² of coordinate differences, then one sqrt (geo and the oracle: |cross / dd| · hypot(dx, dy)).
Every factor is a coordinate difference, at most the diagonal ℓ of the union of the two rows' envelopes and rounded relative to
itself, so cross carries an absolute error of a few u·ℓ·|d| whatever the position of the data, the quotient by |d| an absolute
error of a few u·ℓ, and the divisions, the sqrt and the choice of the minimum among rounded candidates a relative error of a
few u.  Hence
    |got − true| <= K · u · (true + ℓ),   u = 2⁻⁵³.
Measured on the CPU oracle (x86-64, glibc) over every family of tests/pairs_families.py, the largest K a row needs is 0.80
(family D; 0.55 on A, 0.02 on C, 0 on B, whose gaps are computed exactly); DISTANCE_K = 2 leaves a margin of 2.5.  The GPU
maxima are in tests/test_gpu_pairs_exact.py.  A relative tolerance cannot be met where true << ℓ: a point 1e-12 from a
segment between coordinates of 10⁷ has ℓ·u ~ 1e-9 of unavoidable absolute error.  Anything that forms a product of ABSOLUTE coordinates
instead (s.y·dx − p.y·dx) is off by u·|offset|·ℓ and fails it far from the origin.
"""
from __future__ import annotations

from fractions import Fraction as F
from math import isqrt

from oracle import exact

U = 2.0**-53
DISTANCE_K = 2.0

POINTS, CHAINS, AREAS = 0, 1, 2


def _class(kind: str) -> int:
    return {"point": POINTS, "multipoint": POINTS, "linestring": CHAINS, "multilinestring": CHAINS,
            "polygon": AREAS, "multipolygon": AREAS}[kind]


def members(kind: str, row) -> list:
    """the members of a row: points (x, y), chains [coords] or polygons [rings]"""
    if kind in ("point", "linestring", "polygon"):
        return [row]
    return list(row)


def _coords(kind: str, row):
    c = _class(kind)
    for m in members(kind, row):
        if c == POINTS:
            yield m
        elif c == CHAINS:
            yield from m
        else:
            for r in m:
                yield from r


def _scale(*rows) -> int:
    """a power of two that turns every coordinate of the (kind, row) pairs into an integer"""
    den = 1
    for kind, row in rows:
        for x, y in _coords(kind, row):
            den = max(den, F(float(x)).denominator, F(float(y)).denominator)
    return den


def _to_int(kind: str, row, s: int):
    def p(c):
        return (int(F(float(c[0])) * s), int(F(float(c[1])) * s))

    c = _class(kind)
    out = []
    for m in members(kind, row):
        if c == POINTS:
            out.append(p(m))
        elif c == CHAINS:
            out.append([p(q) for q in m])
        else:
            out.append([[p(q) for q in r] for r in m])
    return out


def _closed(ring):
    r = list(ring)
    return r + [r[0]] if r and r[0] != r[-1] else r


# ---- integer chain predicates ---------------------------------------------------------------------------------------------
def _orient(a, b, c) -> int:
    d = (a[0] - c[0]) * (b[1] - c[1]) - (a[1] - c[1]) * (b[0] - c[0])
    return (d > 0) - (d < 0)


def _in_box(p, s, e) -> bool:
    return min(s[0], e[0]) <= p[0] <= max(s[0], e[0]) and min(s[1], e[1]) <= p[1] <= max(s[1], e[1])


def segments_meet(a0, a1, b0, b1) -> bool:
    """closed segments share a point (integer coordinates)"""
    if max(a0[0], a1[0]) < min(b0[0], b1[0]) or max(b0[0], b1[0]) < min(a0[0], a1[0]) or \
            max(a0[1], a1[1]) < min(b0[1], b1[1]) or max(b0[1], b1[1]) < min(a0[1], a1[1]):
        return False
    o1, o2, o3, o4 = _orient(a0, a1, b0), _orient(a0, a1, b1), _orient(b0, b1, a0), _orient(b0, b1, a1)
    if o1 * o2 < 0 and o3 * o4 < 0:
        return True
    return (o1 == 0 and _in_box(b0, a0, a1)) or (o2 == 0 and _in_box(b1, a0, a1)) or \
        (o3 == 0 and _in_box(a0, b0, b1)) or (o4 == 0 and _in_box(a1, b0, b1))


def _segs(chain):
    return list(zip(chain[:-1], chain[1:]))


def chains_meet(a, b) -> bool:
    sb = _segs(b)
    return any(segments_meet(p, q, s, e) for p, q in _segs(a) for s, e in sb)


def point_on_chain(p, chain) -> bool:
    return any(_orient(s, e, p) == 0 and _in_box(p, s, e) for s, e in _segs(chain))


# ---- squared distances -------------------------------------------------------------------------------------------------------
def seg_dist2(p, s, e) -> F:
    """exact squared distance from point p to the closed segment s-e"""
    wx, wy = p[0] - s[0], p[1] - s[1]
    dx, dy = e[0] - s[0], e[1] - s[1]
    dd = dx * dx + dy * dy
    num = wx * dx + wy * dy
    if dd == 0 or num <= 0:
        return F(wx * wx + wy * wy)
    if num >= dd:
        ux, uy = p[0] - e[0], p[1] - e[1]
        return F(ux * ux + uy * uy)
    cross = wx * dy - wy * dx
    return F(cross * cross, dd)


def _pt_chain_d2(p, chain) -> F:
    return min(seg_dist2(p, s, e) for s, e in _segs(chain))


def _chain_chain_d2(a, b) -> F:
    return min(min(_pt_chain_d2(p, a) for p in b), min(_pt_chain_d2(p, b) for p in a))


def _boundary(c: int, m) -> list:
    """the chains bounding a member: [] for a point, [chain] for a chain, the closed rings of a polygon"""
    return [] if c == POINTS else [m] if c == CHAINS else [_closed(r) for r in m]


def _member_intersects(ca, a, cb, b) -> bool:
    if ca > cb:
        ca, a, cb, b = cb, b, ca, a
    if ca == POINTS:
        if cb == POINTS:
            return a == b
        if cb == CHAINS:
            return point_on_chain(a, b)
        return exact.closed_polygon_has(a, b)
    if ca == CHAINS:
        if cb == CHAINS:
            return chains_meet(a, b)
        return any(chains_meet(a, _closed(r)) for r in b) or exact.closed_polygon_has(a[0], b)
    return exact.polygons_intersect(a, b)


def _member_d2(ca, a, cb, b) -> F:
    if _member_intersects(ca, a, cb, b):
        return F(0)
    if ca == POINTS and cb == POINTS:
        return F((a[0] - b[0]) ** 2 + (a[1] - b[1]) ** 2)
    if ca > cb:
        ca, a, cb, b = cb, b, ca, a
    if ca == POINTS:
        return min(_pt_chain_d2(a, r) for r in _boundary(cb, b))
    return min(_chain_chain_d2(x, y) for x in _boundary(ca, a) for y in _boundary(cb, b))


# ---- the operations on float rows ----------------------------------------------------------------------------------------
def intersects(a_row, b_row, kind_a: str, kind_b: str) -> bool:
    s = _scale((kind_a, a_row), (kind_b, b_row))
    ca, cb = _class(kind_a), _class(kind_b)
    A, B = _to_int(kind_a, a_row, s), _to_int(kind_b, b_row, s)
    return any(_member_intersects(ca, x, cb, y) for x in A for y in B)


def distance2(a_row, b_row, kind_a: str, kind_b: str) -> F:
    """exact squared distance (in the units of the input); a row pair without members has none (ValueError)"""
    s = _scale((kind_a, a_row), (kind_b, b_row))
    ca, cb = _class(kind_a), _class(kind_b)
    A, B = _to_int(kind_a, a_row, s), _to_int(kind_b, b_row, s)
    if not A or not B:
        raise ValueError("distance of an empty row")
    best = None
    for x in A:
        for y in B:
            d = _member_d2(ca, x, cb, y)
            best = d if best is None else min(best, d)
            if best == 0:
                return best
    return best / (s * s)


def sqrt_fraction(q: F, bits: int = 160) -> F:
    """sqrt(q) rounded down to `bits` fractional bits: more than 40 significant digits for any distance above 2⁻¹⁰"""
    return F(isqrt(q.numerator * (1 << (2 * bits)) // q.denominator), 1 << bits)


def distance(a_row, b_row, kind_a: str, kind_b: str) -> F:
    return sqrt_fraction(distance2(a_row, b_row, kind_a, kind_b))


def envelope_diagonal(*rows) -> float:
    """ℓ: the diagonal of the union of the envelopes of the (kind, row) pairs"""
    xs, ys = [], []
    for kind, row in rows:
        for x, y in _coords(kind, row):
            xs.append(F(float(x))), ys.append(F(float(y)))
    w, h = max(xs) - min(xs), max(ys) - min(ys)
    return float(sqrt_fraction(w * w + h * h, 80))


def distance_error(got: float, true: F) -> float:
    """|got − true| in doubles (the difference is formed exactly)"""
    return float(abs(F(got) - true))


def distance_bound(true: F, ell: float, k: float = DISTANCE_K) -> float:
    return k * U * (float(true) + ell)


def contains_point(kind_a: str, a_row, p) -> bool:
    s = _scale((kind_a, a_row), ("point", p))
    A, (q,) = _to_int(kind_a, a_row, s), _to_int("point", p, s)
    if _class(kind_a) == AREAS:
        return any(exact.polygon_contains(q, rings) for rings in A)
    if _class(kind_a) != CHAINS:
        raise ValueError("contains_point: (Multi)LineString or (Multi)Polygon rows")
    for c in A:
        if q == c[0] or q == c[-1]:
            if c[0] == c[-1]:
                return True
            continue
        if point_on_chain(q, c):
            return True
    return False


def contains_polygon(kind_a: str, a_row, b_rings) -> bool:
    """(Multi)Polygon a_row contains Polygon b_rings"""
    s = _scale((kind_a, a_row), ("polygon", b_rings))
    return exact.region_contains_polygon(_to_int(kind_a, a_row, s), _to_int("polygon", b_rings, s)[0])
