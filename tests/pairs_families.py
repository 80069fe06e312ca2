"""The row-pair families the row-wise `intersects`, `distance` and `contains` are checked on against tests/pairs_reference.py
(tests/test_pairs_reference_cpu.py: the CPU oracle; tests/test_gpu_pairs_exact.py: the kernels).  Every geometry is VALID.

A  exact translations: rows on a dyadic lattice (integers × 2⁻²⁰ of up to 30 bits, |x| < 2¹⁰) shifted by offsets that are
   multiples of 2⁻²⁰ up to 8.4·10⁶ per axis, so every translated coordinate is exact and every coordinate difference equals
   the origin copy's, while a product of two absolute coordinates needs more than 53 bits and rounds.
B  ulp gaps: a vertex on an edge and 1 or 2 ulps off it on both sides, parallel segments 0 / 1 / 2 ulps apart, collinear
   segments that abut, overlap or leave a 1-ulp gap, a point on / 1 ulp inside / 1 ulp outside an exterior ring and a hole —
   all built with np.nextafter at the final coordinates, at offsets 0, 10³, 6.5·10⁶ and −1.2·10⁷.
C  path-switching lengths: LineString pairs of every combination of lengths in C_LENGTHS, touching, on an edge, 1 ulp apart
   (B's vertices or A's nearest) or apart, in one column; MultiLineString members and unclosed Polygon rings of 31 to 35 coordinates.
D  badly conditioned distances: a point within ulps of a segment 10⁴ long, nearly parallel long segments, a tiny polygon in a
   long hole near both of its ends.

Each case is (kind_a, row_a, kind_b, row_b) in the nesting of GeoArrowArray.from_shapes.
"""
from __future__ import annotations

import zlib

import numpy as np

import shapes

KINDS = shapes.KINDS
SCALE = 131071 * 2.0**-20  # an odd 17-bit multiple of 2⁻²⁰
# multiples of 2⁻²⁰, negative and mixed signs included
A_OFFSETS = [(0.0, 0.0), (1024.0 + 3 * 2.0**-20, -2048.5), (6_500_000.25, 1_234_567.0 + 2.0**-20),
             (-7_654_321.5, 8_123_456.75), (-8_388_607.0 - 5 * 2.0**-20, -8_000_000.0)]
B_OFFSETS = [0.0, 1e3, 6.5e6, -1.2e7]
C_LENGTHS = [0, 1, 2, 3, 16, 31, 32, 33, 34, 35, 64, 200]


def _rng(tag: str):
    return np.random.default_rng(zlib.crc32(tag.encode()))


def _map(row, f):
    """apply f to every coordinate of a nested row"""
    if row is None:
        return None
    if isinstance(row, tuple) and len(row) == 2 and not isinstance(row[0], (list, tuple)):
        return f(row)
    return [_map(r, f) for r in row]


def _dyadic(row):
    """shapes' 0.005-lattice onto integers × 2⁻²⁰: one exact scaling of every lattice point by SCALE / 0.005, so the touching,
    collinear and shared-vertex relations of the lattice rows hold exactly and the coordinates carry up to 30 bits"""
    return _map(row, lambda c: (round(c[0] * 200) * SCALE, round(c[1] * 200) * SCALE))


def translate(row, ox, oy):
    return _map(row, lambda c: (c[0] + ox, c[1] + oy))


# ---- A: valid lattice rows ------------------------------------------------------------------------------------------------------
def _valid_polygon(rng, cx, cy, r, hole):
    ext = shapes.valid_star(rng, cx, cy, r, int(rng.integers(4, 9)))
    if not hole:
        return [ext]
    h = round(float(r) * 0.15, 1) or 0.1
    return [ext, shapes.sq(round(float(cx) - h, 1), round(float(cy) - h, 1), 2 * h)[::-1]]  # a clockwise hole


def _row(rng, kind, i):
    if kind == "point":
        return shapes.random_point(rng)
    if kind == "multipoint":
        return [shapes.random_point(rng) for _ in range(int(rng.integers(1, 4)))]
    if kind == "linestring":
        return shapes.random_linestring(rng)
    if kind == "multilinestring":
        return [shapes.random_linestring(rng) for _ in range(int(rng.integers(1, 3)))]
    cx, cy, r = float(rng.uniform(2, 8)), float(rng.uniform(2, 8)), float(rng.uniform(1, 3))
    if kind == "polygon":
        return _valid_polygon(rng, cx, cy, r, hole=i % 3 == 0)
    # members 2.2 r apart along x: disjoint stars (radii <= r)
    return [_valid_polygon(rng, cx + 2.2 * r * k, cy, r, hole=(i + k) % 4 == 0) for k in range(1 + i % 2)]


def _holes_inside(kind, row):
    """drop a hole that the lattice rounding left touching its exterior (the rows must stay valid)"""
    from oracle import exact

    if kind not in ("polygon", "multipolygon"):
        return row
    fix = [[p[0]] + [h for h in p[1:] if all(exact.ring_position(c, p[0]) == 2 for c in h) and not exact.linestrings_intersect(h, p[0])]
           for p in ([row] if kind == "polygon" else row)]
    return fix[0] if kind == "polygon" else fix


def family_a(ka, kb, n):
    """n valid lattice row pairs of kinds (ka, kb) at the origin; every 4th row of a point or chain side gets a vertex (or an
    edge midpoint) of the other side planted on it"""
    rng = _rng(f"A{ka}x{kb}")
    rb = [_row(rng, kb, i) for i in range(n)]
    ra = [_row(rng, ka, i) for i in range(n)]
    if ka not in ("polygon", "multipolygon"):
        ra = shapes.plant_touching(rng, ka, ra, kb, rb)
    else:
        rb = shapes.plant_touching(rng, kb, rb, ka, ra)
    return [_holes_inside(ka, _dyadic(r)) for r in ra], [_holes_inside(kb, _dyadic(r)) for r in rb]


def family_a_contains(n):
    """(Multi)Polygon x Polygon pairs for contains: shapes.contains_cases on the dyadic lattice, as Polygon rows"""
    A, B = shapes.contains_cases(_rng("Acontains"), n_random=n)
    return [_dyadic(a) for a in A], [_dyadic(b) for b in B]


# ---- B: ulp gaps ----------------------------------------------------------------------------------------------------------------
def _up(x, k):
    for _ in range(abs(k)):
        x = float(np.nextafter(x, np.inf if k > 0 else -np.inf))
    return x


def _sq(x, y, s):
    return [(x, y), (x + s, y), (x + s, y + s), (x, y + s), (x, y)]


def _lift(kind, m, o):
    """the primitive member m as a row of `kind`; Multi* rows get a far member FIRST, so the near one is the last member"""
    far = -40.0 + o
    if kind in ("point", "linestring", "polygon"):
        return m
    if kind == "multipoint":
        return [(far, far), m]
    if kind == "multilinestring":
        return [[(far, far), (far + 1, far)], m]
    return [[_sq(far, far, 1.0)], m]


def _prim_cases(o):
    """primitive (class_a, member_a, class_b, member_b) cases at offset o; classes 'p', 'l', 'a'"""
    o += 16.0  # local coordinates in [16, 32): no coordinate near 0, where an ulp is subnormal
    out = []
    # exterior [o, o+8]², clockwise hole [o+2, o+6]²; a slope-1/2 edge from (o, o) to (o+8, o+4) as a chain
    ext = _sq(o, o, 8.0)
    hole = _sq(o + 2, o + 2, 4.0)[::-1]
    poly = [ext, hole]
    diag = [(o, o), (o + 8, o + 4)]
    horiz = [(o, o + 1), (o + 4, o + 1)]
    for k in (-2, -1, 0, 1, 2):
        # a vertex on / k ulps off an axis-aligned and a dyadic-slope edge
        out.append(("p", (o + 1.5, _up(o + 1, k)), "l", horiz))
        out.append(("p", (o + 4, _up(o + 2, k)), "l", diag))
        out.append(("p", (_up(o + 4, k), o + 2), "l", diag))
        # a chain vertex touching an edge from one side: the chain leaves the edge away from it
        out.append(("l", [(o + 2, _up(o + 1, k)), (o + 3, o + 5)], "l", horiz))
        out.append(("l", [(o + 6, _up(o + 3, k)), (o + 5, o + 7)], "l", diag))
        # a point on / off the exterior ring (x = o + 8) and on / off the hole ring (x = o + 2)
        out.append(("p", (_up(o + 8, k), o + 3), "a", poly))
        out.append(("p", (_up(o + 2, k), o + 4), "a", poly))
        # a chain ending on / off the exterior from outside, on / off the hole from inside the hole
        out.append(("l", [(o + 10, o + 3), (_up(o + 8, k), o + 3)], "a", poly))
        out.append(("l", [(o + 4, o + 4), (_up(o + 2, k), o + 4.5)], "a", poly))
        # a polygon corner on / off the exterior from outside and on / off the hole edge from inside the hole
        out.append(("a", [[(_up(o + 8, k), o + 3), (o + 10, o + 2), (o + 10, o + 4), (_up(o + 8, k), o + 3)]], "a", poly))
        out.append(("a", [[(_up(o + 2, k), o + 4), (o + 3, o + 3.5), (o + 3, o + 4.5), (_up(o + 2, k), o + 4)]], "a", poly))
        # a triangle corner on / off a slope-1/2 edge of a triangle, from below
        tri = [[(o, o), (o + 8, o + 4), (o, o + 4), (o, o)]]
        out.append(("a", [[(o + 4, _up(o + 2, k)), (o + 5, o), (o + 6, o + 1), (o + 4, _up(o + 2, k))]], "a", tri))
    for k in (0, 1, 2):
        # parallel segments k ulps apart, horizontal and slope 1/2 (each endpoint moved k ulps)
        out.append(("l", [(o + 1, _up(o + 1, k)), (o + 5, _up(o + 1, k))], "l", horiz))
        out.append(("l", [(o + 2, _up(o + 1, k)), (o + 10, _up(o + 5, k))], "l", diag))
        # a polygon edge parallel to the exterior's bottom edge, k ulps below it
        out.append(("a", [[(o + 1, _up(o, -k)), (o + 3, _up(o, -k)), (o + 3, o - 2), (o + 1, o - 2), (o + 1, _up(o, -k))]], "a", poly))
    for start in ("abut", "overlap", "gap1", "gap2"):
        x = {"abut": o + 4, "overlap": o + 3, "gap1": _up(o + 4, 1), "gap2": _up(o + 4, 2)}[start]
        out.append(("l", [(x, o + 1), (o + 7, o + 1)], "l", horiz))  # collinear with horiz, which ends at x = o + 4
        out.append(("l", [(x, o + 1), (o + 7, o + 1)], "a", [_sq(o, o - 1, 4.0)]))  # from on / inside / right of its right side
    return out


def family_b():
    """the ulp-gap cases over every type pair with a chain or polygon side, at every B offset"""
    cls_kinds = {"p": ("point", "multipoint"), "l": ("linestring", "multilinestring"), "a": ("polygon", "multipolygon")}
    cases = []
    for o in B_OFFSETS:
        for ca, ma, cb, mb in _prim_cases(o):
            for ka in cls_kinds[ca]:
                for kb in cls_kinds[cb]:
                    cases.append((ka, _lift(ka, ma, o), kb, _lift(kb, mb, o), o))
                    cases.append((kb, _lift(kb, mb, o), ka, _lift(ka, ma, o), o))
    return cases


def family_b_contains_point():
    """(Multi)Polygon / (Multi)LineString x Point on / 1 ulp off rings, holes and chain ends"""
    out = []
    for o in (b + 16.0 for b in B_OFFSETS):
        poly = [_sq(o, o, 8.0), _sq(o + 2, o + 2, 4.0)[::-1]]
        open_l = [(o, o + 1), (o + 4, o + 1), (o + 8, o + 5)]
        closed_l = [(o, o), (o + 4, o), (o + 4, o + 2), (o, o)]
        for k in (-1, 0, 1):
            for p in [(_up(o + 8, k), o + 3), (_up(o + 2, k), o + 4), (o + 4, _up(o + 6, k))]:
                out += [("polygon", poly, p), ("multipolygon", [[_sq(o - 40, o - 40, 1.0)], poly], p)]
            for p in [(o + 2, _up(o + 1, k)), (_up(o, k), o + 1), (o + 6, _up(o + 3, k)), (_up(o + 8, k), o + 5), (_up(o, k), o)]:
                for line in (open_l, closed_l):
                    out += [("linestring", line, p), ("multilinestring", [[(o - 40, o - 40), (o - 39, o - 40)], line], p)]
    return out


def family_b_contains_polygon():
    """(Multi)Polygon x Polygon sharing a boundary edge, and 1 ulp in / out of it"""
    out = []
    for o in (b + 16.0 for b in B_OFFSETS):
        big = [_sq(o, o, 8.0)]
        for k in (-1, 0, 1):
            b = [[(o, o), (o + 4, o), (o + 4, o + 4), (_up(o, k), o + 4), (o, o)]]  # shares the bottom edge, left side k ulps off
            out += [("polygon", big, b), ("multipolygon", [[_sq(o - 40, o - 40, 1.0)], big], b)]
            out.append(("polygon", [_sq(o, o, 8.0), _sq(o + 2, o + 2, 4.0)[::-1]], [_sq(_up(o + 2, k), o + 2, 2.0)]))  # at the hole
    return out


# ---- C: lengths at the path switches ------------------------------------------------------------------------------------------
C_MODES = ["touch", "on_edge", "ulp", "flat_ulp", "apart"]


def family_c(o=6.5e6):
    """LineString x LineString over every (len_a, len_b) in C_LENGTHS² and every mode of C_MODES, in one column.  A zigzags
    along x (step 1/2) between y = 0 and its peaks y = 1/4 on odd vertices; B zigzags above it between its troughs on odd
    vertices and 1/4 higher.  touch: B's troughs on A's peaks; ulp: 1 ulp above them; apart: 1/2 above them; on_edge: B's first
    trough on the midpoint of A's first segment, the others 1/2 above A's peaks; flat_ulp: B is straight, 1 ulp above A's
    peaks, with its vertices half-way between them (the nearest pairs are A's vertices against B's segments)"""
    rows = []
    for la in C_LENGTHS:
        for lb in C_LENGTHS:
            for mode in C_MODES:
                a = [(o + 0.5 * i, o + (0.25 if i % 2 else 0.0)) for i in range(la)]
                trough = {"touch": o + 0.25, "ulp": _up(o + 0.25, 1), "apart": o + 0.75, "on_edge": o + 0.75, "flat_ulp": 0.0}[mode]
                b = [(o + 0.5 * i, trough if i % 2 else trough + 0.25) for i in range(lb)]
                if mode == "flat_ulp":
                    b = [(o + 0.25 + 0.5 * i, _up(o + 0.25, 1)) for i in range(lb)]
                if mode == "on_edge" and lb > 1:
                    b[1] = (o + 0.25, o + 0.125)  # the midpoint of A's first segment (o, o) - (o + 1/2, o + 1/4)
                rows.append(("linestring", a, "linestring", b))
    return rows


def _parabola_ring(n, o, x0=0.0, closed=False):
    """a strictly convex ring of n distinct vertices (i/8, i²/64) + (x0, 0); closed: the first vertex repeated at the end"""
    pts = [(o + x0 + i / 8.0, o + i * i / 64.0) for i in range(n)]
    return pts + [pts[0]] if closed else pts


def family_c_rings(o=6.5e6):
    """Polygon and MultiLineString rows whose rings / members have 31 to 35 coordinates, against a LineString that touches,
    crosses 1 ulp short of, or misses the CLOSING edge of an unclosed ring (the chord from the last vertex back to the first)"""
    rows = []
    for n in (31, 32, 33, 34, 35):
        for closed in (False, True):
            ring = _parabola_ring(n - (1 if closed else 0), o, closed=closed)
            last = ring[-2] if closed else ring[-1]
            # the chord's midpoint is exact (both ends on the lattice)
            mx, my = (ring[0][0] + last[0]) / 2, (ring[0][1] + last[1]) / 2
            for k in (0, 1, 4096):
                # a segment from above-left ending on / k ulps above the chord's midpoint (the chord has slope > 0)
                tip = (mx, _up(my, k))
                line = [(mx - 1.0, my + 3.0), tip]
                rows.append(("polygon", [ring], "linestring", line))
                rows.append(("linestring", line, "polygon", [ring]))
                rows.append(("multilinestring", [ring[:n], [(o - 40, o - 40), (o - 39, o - 40)]], "linestring", line))
    return rows


# ---- D: badly conditioned distances -------------------------------------------------------------------------------------------
def family_d():
    out = []
    for o in (0.0, 6.5e6, -1.2e7):
        seg = [(o, o), (o + 8192.0, o + 4096.0)]
        for k in (1, 2, 3, 7, 1000):
            out.append(("point", (o + 4096.0, _up(o + 2048.0, k)), "linestring", seg))
            out.append(("point", (o + 4096.0 + 1e-12 * k, o + 2048.0), "linestring", seg))
            # nearly parallel long segments: B's far end k ulps above A's line
            out.append(("linestring", [(o + 1.0, _up(o + 0.5, 1)), (o + 8190.0, _up(o + 4095.0, k))], "linestring", seg))
        # a 1e-3 square inside a long thin hole, near each end of it
        ext = _sq(o - 10.0, o - 10.0, 10020.0)
        hole = [(o, o), (o, o + 1.0), (o + 10000.0, o + 1.0), (o + 10000.0, o), (o, o)]
        for x in (o + 1e-6, o + 9999.998):
            for y in (o + 1e-9, o + 0.5):
                tiny = [(x, y), (x + 1e-3, y), (x + 1e-3, y + 1e-3), (x, y + 1e-3), (x, y)]
                out.append(("polygon", [ext, hole], "polygon", [tiny]))
                out.append(("linestring", tiny[:3], "polygon", [ext, hole]))
                out.append(("point", (x, y), "polygon", [ext, hole]))
    return out
