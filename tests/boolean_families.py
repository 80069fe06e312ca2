"""The (Multi)Polygon row pairs `intersection_area` and the boolean ops are checked on far from the origin, at ulp-scale gaps
and at the ring lengths where the lane grouping of the node and overlap passes switches (tests/test_boolean_families_cpu.py:
the referees; tests/test_gpu_boolean_families.py: the kernels).  Every operand row is VALID.  Each case is
(kind_a, row_a, kind_b, row_b, tag) in the nesting of GeoArrowArray.from_shapes; `members(kind, row)` gives the referees' form.

BA  exact translations: pairs_families.family_a over polygon / multipolygon in both orders, shifted by every A_OFFSETS entry.
BB  ulp gaps: the polygon x polygon cases of pairs_families.family_b, and sub-ulp cases at every B_OFFSETS entry — a triangle
    tip 1 or 2 ulps across (or 1 ulp short of) an axis-aligned edge, a slope-1/2 edge and a hole's edge, with tip edges of
    slope 1/2, 1/64 and 2⁻²⁰; combs of 2 to 8 teeth whose tips cross one edge with crossings about 0, 1 and 2 ulps apart; an
    edge passing on / 1 ulp beside a corner; two edges crossing at an angle of 2⁻³⁰.  All four column-type combinations, both
    operand orders.  Where two constructed crossings lie within half an ulp of each other they round to one point, which the
    assembler must resolve (DESIGN.md §4.19, the spike and pinch rule).
BC  ring lengths: strictly convex dyadic rings on the parabola y = x² at offset 6.5·10⁶ of every length in BC_LENGTHS (edges),
    vertices of the two operands interleaved so that the rings cross about twice per edge; each length against a 5-edge
    partner in both roles, the diagonal (n, n), the same lengths as a hole the partner crosses, and 200 against 5 once.
    Every row closed and unclosed.
BD  analytic answers: two combs of k teeth crossing in a k x k grid, 40 lattice squares against a rectangle, a square with 40
    holes against a rectangle; dyadic coordinates with power-of-two edge spans wherever edges cross, so every crossing
    point is exact; the expected rings of all three ops in closed form.
"""
from __future__ import annotations

import pairs_families as PF

POLY_KINDS = ("polygon", "multipolygon")
OPS = ("intersection", "union", "difference")
BC_LENGTHS = [3, 4, 5, 7, 8, 9, 15, 16, 17, 31, 32, 33, 63, 64, 65]
BC_OFFSET = 6.5e6
BD_K = [1, 31, 32, 33, 100]


def members(kind, row):
    return [row] if kind == "polygon" else row


def swap(c):
    return (c[2], c[3], c[0], c[1], c[4])


# ---- BA ---------------------------------------------------------------------------------------------------------------------
def family_ba(n=24):
    """(origin cases, {offset: translated cases}) — the same cases in the same order at every offset"""
    base = []
    for ka in POLY_KINDS:
        for kb in POLY_KINDS:
            ra, rb = PF.family_a(ka, kb, n)
            for i, (a, b) in enumerate(zip(ra, rb)):
                base.append((ka, a, kb, b, f"BA {ka}x{kb} {i}"))
                base.append((kb, b, ka, a, f"BA {kb}x{ka} {i} swapped"))
    moved = {(ox, oy): [(c[0], PF.translate(c[1], ox, oy), c[2], PF.translate(c[3], ox, oy), c[4]) for c in base]
             for ox, oy in PF.A_OFFSETS[1:]}
    return base, moved


# ---- BB ---------------------------------------------------------------------------------------------------------------------
SLOPES = {"1/2": 0.5, "1/64": 1 / 64, "2^-20": 2.0**-20}


def _tri_tip_x(o, x_edge, k, side, s):
    """a triangle pointing along -side·x whose tip is k ulps past the vertical line x = x_edge (k < 0: short of it), tip edges
    of slope ±s over a run of 2"""
    tip = PF._up(x_edge, -side * k)
    base = x_edge + 2.0 * side
    return [(tip, o + 3), (base, o + 3 - 2 * s), (base, o + 3 + 2 * s), (tip, o + 3)]


def _sub_ulp_prims(o):
    """(tag, A member, B member) at offset o; A members are polygons (lists of rings)"""
    o += 16.0  # local coordinates in [16, 32)
    sq = PF._sq
    square = [sq(o, o, 8.0)]
    holed = [sq(o, o, 8.0), sq(o + 2, o + 2, 4.0)[::-1]]
    tri = [[(o, o), (o + 8, o + 4), (o, o + 4), (o, o)]]  # the slope-1/2 edge (o, o) - (o + 8, o + 4), interior above
    out = []
    for sname, s in SLOPES.items():
        for k in (1, 2, -1):
            what = f"{k} ulp across" if k > 0 else "1 ulp short"
            # from outside the exterior across x = o + 8 (B to the right, pointing left)
            out.append((f"tip {what} exterior edge, slope {sname}", square, [_tri_tip_x(o, o + 8, k, 1, s)]))
            # from inside the hole across its edge x = o + 6 (B inside the hole, pointing right)
            t = [(PF._up(o + 6, k), o + 4), (o + 4, o + 4 + 2 * s), (o + 4, o + 4 - 2 * s), (PF._up(o + 6, k), o + 4)]
            out.append((f"tip {what} hole edge, slope {sname}", holed, [t]))
            # from below across the slope-1/2 edge at (o + 4, o + 2): tip edges at slope 1/2 -+ s
            ty = PF._up(o + 2, k)
            t = [(o + 4, ty), (o + 2, o + 1 - 2 * s), (o + 6, o + 3 - 2 * s), (o + 4, ty)]
            out.append((f"tip {what} slope-1/2 edge, relative slope {sname}", tri, [t]))
    # combs: n teeth from a bar right of x = o + 8, tips 1 ulp across it, tooth edges of slope m: crossings ≈ 2m ulps apart
    for n in (2, 3, 5, 8):
        for gap, m in ((0, 2.0**-20), (1, 0.5), (2, 1.0)):
            tip = PF._up(o + 8, -1)
            w = 0.25 * m  # half-width of a tooth at its base (run 1/4)
            ring = [(o + 9, o + 0.5), (o + 9, o + 7.5), (o + 8.25, o + 7.5)]
            for i in reversed(range(n)):
                yc = o + 1 + 0.75 * i
                ring += [(o + 8.25, yc + w), (tip, yc), (o + 8.25, yc - w)]
            ring += [(o + 8.25, o + 0.5), (o + 9, o + 0.5)]
            out.append((f"comb {n} teeth, crossings ~{gap} ulps apart", square, [ring]))
    # an edge of slope -1 through / 1 ulp beside the corner (o + 8, o + 8), B to the upper right
    for k in (-1, 0, 1):
        t = [(o + 6, PF._up(o + 10, k)), (o + 10, PF._up(o + 6, k)), (o + 10, o + 10), (o + 6, PF._up(o + 10, k))]
        out.append((f"edge {k} ulp beside a corner", square, [t]))
    # a thin wedge: B's edge crosses A's bottom edge at (o + 4, o) at an angle of 2^-30
    for d in (2.0**-29, 2.0**-28):
        t = [(o + 2, o - d), (o + 6, o + d), (o + 6, o - 1), (o + 2, o - d)]
        out.append((f"thin wedge, rise {d:g}", square, [t]))
    return out


def family_bb():
    """the polygon x polygon cases of pairs_families.family_b, then the sub-ulp cases in every column-type combination and both
    operand orders, at every B offset"""
    cases = [(c[0], c[1], c[2], c[3], f"B family_b {i} @{c[4]}") for i, c in enumerate(PF.family_b())
             if c[0] in POLY_KINDS and c[2] in POLY_KINDS]
    for o in PF.B_OFFSETS:
        for tag, ma, mb in _sub_ulp_prims(o):
            for ka in POLY_KINDS:
                for kb in POLY_KINDS:
                    c = (ka, PF._lift(ka, ma, o), kb, PF._lift(kb, mb, o), f"BB {tag} @{o} {ka}x{kb}")
                    cases += [c, swap(c)]
    return cases


# ---- BC ---------------------------------------------------------------------------------------------------------------------
def _cup(xs, o, closed):
    """a strictly convex ring on y = x² through the given dyadic x (increasing), shifted by (o, o)"""
    pts = [(o + x, o + x * x) for x in xs]
    return pts + [pts[0]] if closed else pts


def _ring_n(n, o, closed):
    """n vertices at x = i/8"""
    return _cup([i / 8.0 for i in range(n)], o, closed)


def _ring_interleaved(n, o, closed):
    """n vertices at x = (2i + 1)/16, between those of _ring_n"""
    return _cup([(2 * i + 1) / 16.0 for i in range(n)], o, closed)


def _partner5(n, o, closed):
    """5 vertices spread over the x range of _ring_n(n), off its vertices (multiples of 2^-12, so y = x² is exact)"""
    span = (n - 1) / 8.0
    xs = [round(span * (2 * k + 1) / 10.0 * 4096 + 1) / 4096.0 for k in range(5)]
    return _cup(xs, o, closed)


def _holed(ring, o):
    """a square around the parabola ring with that ring as its hole"""
    xs, ys = [p[0] for p in ring], [p[1] for p in ring]
    x0, y0 = min(xs) - 1.0, min(ys) - 1.0
    s = max(max(xs) - x0, max(ys) - y0) + 1.0
    return [PF._sq(x0, y0, s), ring[::-1]]


def _unclosed(row):
    """the row with the closing coordinate of every ring dropped (Chain closes it again)"""
    return [r[:-1] for r in row]


def family_bc(o=BC_OFFSET):
    """(closed cases, the same cases unclosed); Polygon x Polygon"""
    rows = []
    for n in BC_LENGTHS:
        a, b5 = _ring_n(n, o, True), _partner5(n, o, True)
        rows.append(("polygon", [a], "polygon", [b5], f"BC {n} x 5"))
        rows.append(("polygon", [b5], "polygon", [a], f"BC 5 x {n}"))
        rows.append(("polygon", [a], "polygon", [_ring_interleaved(n, o, True)], f"BC {n} x {n}"))
        rows.append(("polygon", _holed(a, o), "polygon", [b5], f"BC hole {n} x 5"))
        rows.append(("polygon", [b5], "polygon", _holed(a, o), f"BC 5 x hole {n}"))
    rows.append(("polygon", [_ring_n(200, o, True)], "polygon", [_partner5(200, o, True)], "BC 200 x 5"))
    return rows, [(c[0], _unclosed(c[1]), c[2], _unclosed(c[3]), c[4] + " unclosed") for c in rows]


# ---- BD ---------------------------------------------------------------------------------------------------------------------
def _rect_ccw(x0, y0, x1, y1):
    return [(x0, y0), (x1, y0), (x1, y1), (x0, y1), (x0, y0)]


def _rect_cw(x0, y0, x1, y1):
    return [(x0, y0), (x0, y1), (x1, y1), (x1, y0), (x0, y0)]


def _w(k):
    w = 1.0
    while w < 2 * k + 1:
        w *= 2
    return w


def comb(k):
    """k horizontal teeth [0, W] x [2i + 1/2, 2i + 1] on a spine [-W, 0] x [1/2, 2k - 1] (W the power of two >= 2k + 1): every
    edge a crossing can lie on spans W or 2W"""
    W = _w(k)
    r = [(-W, 0.5)]
    for i in range(k):
        r += [(W, 2 * i + 0.5), (W, 2 * i + 1.0)]
        if i < k - 1:
            r += [(0.0, 2 * i + 1.0), (0.0, 2 * i + 2.5)]
    r += [(-W, 2 * k - 1.0), (-W, 0.5)]
    return [r]


def transpose(poly):
    return [[(y, x) for x, y in ring] for ring in poly]


def combs_expected(k):
    """A = comb(k), B = its transpose: {op: members} in the output form of gpl_boolean_op"""
    W = _w(k)
    inter = [[_rect_ccw(2 * j + 0.5, 2 * i + 0.5, 2 * j + 1.0, 2 * i + 1.0)] for j in range(k) for i in range(k)]
    # union: one shell, holes between the teeth, left of B's first tooth and below A's first tooth
    s = [(-W, 0.5), (0.5, 0.5), (0.5, -W), (2 * k - 1.0, -W)]
    for i in range(k):
        s += [(2 * k - 1.0, 2 * i + 0.5), (W, 2 * i + 0.5), (W, 2 * i + 1.0), (2 * k - 1.0, 2 * i + 1.0)]
    for j in reversed(range(k)):
        s += [(2 * j + 1.0, W), (2 * j + 0.5, W), (2 * j + 0.5, 2 * k - 1.0)]
        if j > 0:
            s.append((2 * j - 1.0, 2 * k - 1.0))
    s += [(-W, 2 * k - 1.0), (-W, 0.5)]
    holes = [_rect_cw(2 * j + 1.0, 2 * i + 1.0, 2 * j + 2.5, 2 * i + 2.5) for i in range(k - 1) for j in range(k - 1)]
    holes += [_rect_cw(0.0, 2 * i + 1.0, 0.5, 2 * i + 2.5) for i in range(k - 1)]
    holes += [_rect_cw(2 * j + 1.0, 0.0, 2 * j + 2.5, 0.5) for j in range(k - 1)]
    union = [[s] + sorted(holes)]
    # difference: the spine with stubs [0, 1/2] of the teeth, and the pieces of each tooth between and beyond B's teeth
    sp = [(-W, 0.5)]
    for i in range(k):
        sp += [(0.5, 2 * i + 0.5), (0.5, 2 * i + 1.0)]
        if i < k - 1:
            sp += [(0.0, 2 * i + 1.0), (0.0, 2 * i + 2.5)]
    sp += [(-W, 2 * k - 1.0), (-W, 0.5)]
    pieces = [[_rect_ccw(2 * j + 1.0, 2 * i + 0.5, 2 * j + 2.5, 2 * i + 1.0)] for i in range(k) for j in range(k - 1)]
    pieces += [[_rect_ccw(2 * k - 1.0, 2 * i + 0.5, W, 2 * i + 1.0)] for i in range(k)]
    diff = [[sp]] + sorted(pieces, key=lambda m: m[0][0])
    area_a = W * (2 * k - 1.5) + k * W * 0.5
    return {"intersection": sorted(inter, key=lambda m: m[0][0]), "union": union, "difference": diff}, area_a, k * k / 4.0


def squares_expected():
    """A: 40 unit squares at (2i, 2j), i < 8, j < 5, as one MultiPolygon; B: [5/2, 16] x [-1, 16], which covers the squares
    with i >= 2 and cuts those with i = 1 at x = 5/2"""
    A = [[PF._sq(2.0 * i, 2.0 * j, 1.0)] for i in range(8) for j in range(5)]
    B = [_rect_ccw(2.5, -1.0, 16.0, 16.0)]
    inter = [[_rect_ccw(2.5, 2.0 * j, 3.0, 2.0 * j + 1.0)] for j in range(5)]
    inter += [[PF._sq(2.0 * i, 2.0 * j, 1.0)] for i in range(2, 8) for j in range(5)]
    s = [(2.0, 0.0), (2.5, 0.0), (2.5, -1.0), (16.0, -1.0), (16.0, 16.0), (2.5, 16.0)]
    for j in reversed(range(1, 5)):
        s += [(2.5, 2.0 * j + 1.0), (2.0, 2.0 * j + 1.0), (2.0, 2.0 * j), (2.5, 2.0 * j)]
    s += [(2.5, 1.0), (2.0, 1.0), (2.0, 0.0)]
    union = [[PF._sq(0.0, 2.0 * j, 1.0)] for j in range(5)] + [[s]]
    diff = [[PF._sq(0.0, 2.0 * j, 1.0)] for j in range(5)] + [[_rect_ccw(2.0, 2.0 * j, 2.5, 2.0 * j + 1.0)] for j in range(5)]
    exp = {"intersection": sorted(inter, key=lambda m: m[0][0]), "union": union, "difference": sorted(diff, key=lambda m: m[0][0])}
    return A, B, exp, 40.0, 35.0 - 2.5


def holes_expected():
    """A: [0, 16] x [0, 10] with 40 unit holes at (2i + 1/2, 2j + 1/2); B: [3, 20] x [-1, 11], which covers the holes with
    i >= 2 and cuts those with i = 1 at x = 3"""
    A = [_rect_ccw(0.0, 0.0, 16.0, 10.0)] + [_rect_cw(2 * i + 0.5, 2 * j + 0.5, 2 * i + 1.5, 2 * j + 1.5) for i in range(8) for j in range(5)]
    B = [_rect_ccw(3.0, -1.0, 20.0, 11.0)]
    s = [(3.0, 0.0), (16.0, 0.0), (16.0, 10.0), (3.0, 10.0)]
    for j in reversed(range(5)):
        s += [(3.0, 2 * j + 1.5), (3.5, 2 * j + 1.5), (3.5, 2 * j + 0.5), (3.0, 2 * j + 0.5)]
    s.append((3.0, 0.0))
    inter = [[s] + sorted(_rect_cw(2 * i + 0.5, 2 * j + 0.5, 2 * i + 1.5, 2 * j + 1.5) for i in range(2, 8) for j in range(5))]
    u = [(0.0, 0.0), (3.0, 0.0), (3.0, -1.0), (20.0, -1.0), (20.0, 11.0), (3.0, 11.0), (3.0, 10.0), (0.0, 10.0), (0.0, 0.0)]
    uh = [_rect_cw(0.5, 2 * j + 0.5, 1.5, 2 * j + 1.5) for j in range(5)] + [_rect_cw(2.5, 2 * j + 0.5, 3.0, 2 * j + 1.5) for j in range(5)]
    union = [[u] + sorted(uh)]
    d = [(0.0, 0.0), (3.0, 0.0)]
    for j in range(5):
        d += [(3.0, 2 * j + 0.5), (2.5, 2 * j + 0.5), (2.5, 2 * j + 1.5), (3.0, 2 * j + 1.5)]
    d += [(3.0, 10.0), (0.0, 10.0), (0.0, 0.0)]
    diff = [[d] + sorted(_rect_cw(0.5, 2 * j + 0.5, 1.5, 2 * j + 1.5) for j in range(5))]
    return A, B, {"intersection": inter, "union": union, "difference": diff}, 160.0 - 40.0, 13 * 10.0 - 30.0 - 2.5


def family_bd(ks=BD_K):
    """[(kind_a, row_a, kind_b, row_b, tag, {op: expected members}, exact intersection area)]"""
    out = []
    for k in ks:
        exp, _, inter = combs_expected(k)
        out.append(("polygon", comb(k), "polygon", transpose(comb(k)), f"BD combs {k}", exp, inter))
    A, B, exp, _, inter = squares_expected()
    out.append(("multipolygon", A, "polygon", B, "BD 40 squares", exp, inter))
    A, B, exp, _, inter = holes_expected()
    out.append(("polygon", A, "polygon", B, "BD 40 holes", exp, inter))
    return out
