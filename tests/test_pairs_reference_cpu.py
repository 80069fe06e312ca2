"""CPU tests of tests/pairs_reference.py, the exact referee of the row-wise pair operations: its answers on hand-worked cases,
the CPU oracle (geo's arithmetic) against it on every family of tests/pairs_families.py — booleans equal, distances within
the bound stated in pairs_reference — and the oracle bit-identical under exact translation.  No GPU needed."""
from decimal import Decimal, getcontext
from fractions import Fraction as F

import numpy as np
import pytest

import pairs_families as PF
import pairs_reference as R
from geopolars_b200 import GeoArrowArray, GeometryType

T = {k: GeometryType[k.upper()] for k in PF.KINDS}


def sq(x, y, s):
    return [(x, y), (x + s, y), (x + s, y + s), (x, y + s), (x, y)]


# ---- the referee on hand-worked answers -------------------------------------------------------------------------------------
def test_point_segment_cases():
    seg = [(0.0, 0.0), (10.0, 0.0)]
    assert R.distance2((-3.0, 4.0), seg, "point", "linestring") == 25  # r <= 0: to the start
    assert R.distance2((5.0, 3.0), seg, "point", "linestring") == 9  # interior: perpendicular
    assert R.distance2((13.0, -4.0), seg, "point", "linestring") == 25  # r >= 1: to the end
    assert R.distance2((10.0, 0.0), seg, "point", "linestring") == 0 and R.intersects((10.0, 0.0), seg, "point", "linestring")
    # a slope-1/2 segment: the perpendicular foot is interior, cross = 2·4 - 1·3 = 5 over |d|² = 5
    assert R.distance2((3.0, 4.0), [(0.0, 0.0), (4.0, 2.0)], "point", "linestring") == F(25, 5)
    # sqrt to 40 digits
    getcontext().prec = 60
    got = R.distance((1.0, 1.0), (0.0, 0.0), "point", "point")
    assert abs(Decimal(got.numerator) / Decimal(got.denominator) - Decimal(2).sqrt()) < Decimal(10) ** -45


def test_holes_touching_overlap_and_members():
    poly = [sq(0.0, 0.0, 10.0), sq(2.0, 2.0, 6.0)[::-1]]
    assert not R.intersects((4.0, 5.0), poly, "point", "polygon")
    assert R.distance2((4.0, 5.0), poly, "point", "polygon") == 4  # in the hole: to the hole's side x = 2
    assert R.distance2(poly, [(4.0, 4.0), (5.0, 6.0)], "polygon", "linestring") == 4  # a line in the hole
    assert R.distance2(poly, [sq(4.0, 4.0, 1.0)], "polygon", "polygon") == 4
    assert R.distance2(poly, (12.0, 5.0), "polygon", "point") == 4  # outside: to the exterior
    assert R.intersects(poly, (2.0, 5.0), "polygon", "point") and R.intersects(poly, (1.0, 5.0), "polygon", "point")
    # touching at a vertex only
    assert R.intersects([sq(0.0, 0.0, 1.0)], [sq(1.0, 1.0, 1.0)], "polygon", "polygon")
    assert R.distance2([sq(0.0, 0.0, 1.0)], [sq(1.0, 1.0, 1.0)], "polygon", "polygon") == 0
    # collinear segments: overlapping, abutting, 1 apart
    a = [(0.0, 0.0), (2.0, 0.0)]
    assert R.intersects(a, [(1.0, 0.0), (3.0, 0.0)], "linestring", "linestring")
    assert R.intersects(a, [(2.0, 0.0), (3.0, 0.0)], "linestring", "linestring")
    assert R.distance2(a, [(3.0, 0.0), (4.0, 0.0)], "linestring", "linestring") == 1
    # a Multi* row whose nearest member is the last one
    assert R.distance2([(100.0, 100.0), (50.0, 50.0), (3.0, 4.0)], (0.0, 0.0), "multipoint", "point") == 25
    mls = [[(100.0, 0.0), (100.0, 5.0)], [(6.0, -1.0), (6.0, 1.0)]]
    assert R.distance2(mls, [(0.0, 0.0), (1.0, 0.0)], "multilinestring", "linestring") == 25
    mpoly = [[sq(50.0, 50.0, 1.0)], [sq(3.0, 0.0, 1.0)]]
    assert R.distance2(mpoly, (0.0, 0.5), "multipolygon", "point") == 9
    # 1 ulp at 6.5e6: no intersection, the exact gap
    o = 6.5e6
    up = float(np.nextafter(o + 1.0, np.inf))
    assert not R.intersects([(o, o + 1.0), (o + 4, o + 1.0)], [(o + 1, up), (o + 2, up)], "linestring", "linestring")
    assert R.distance2([(o, o + 1.0), (o + 4, o + 1.0)], [(o + 1, up), (o + 2, up)], "linestring", "linestring") == F(up - o - 1) ** 2


def test_contains_semantics():
    big = [sq(0.0, 0.0, 10.0)]
    assert R.contains_polygon("polygon", big, [sq(0.0, 0.0, 5.0)])  # shares two boundary edges
    assert R.contains_polygon("polygon", big, big)
    assert not R.contains_polygon("polygon", big, [sq(5.0, 5.0, 10.0)])
    assert not R.contains_polygon("polygon", [big[0], sq(4.0, 4.0, 2.0)[::-1]], [sq(4.0, 4.0, 2.0)])  # is the hole
    assert R.contains_polygon("multipolygon", [[sq(20.0, 0.0, 1.0)], big], [sq(1.0, 1.0, 2.0)])
    assert R.contains_point("polygon", big, (5.0, 5.0)) and not R.contains_point("polygon", big, (10.0, 5.0))
    open_l, closed_l = [(0.0, 0.0), (2.0, 0.0), (2.0, 2.0)], [(0.0, 0.0), (2.0, 0.0), (2.0, 2.0), (0.0, 0.0)]
    assert not R.contains_point("linestring", open_l, (0.0, 0.0))  # an end point of an open line is its boundary
    assert R.contains_point("linestring", open_l, (2.0, 0.0)) and R.contains_point("linestring", open_l, (2.0, 1.0))
    assert R.contains_point("linestring", closed_l, (0.0, 0.0)) and R.contains_point("linestring", closed_l, (1.0, 1.0))
    assert R.contains_point("multilinestring", [open_l, [(-1.0, 0.0), (1.0, 0.0)]], (0.0, 0.0))


def test_integer_segment_predicate_matches_exact_py():
    """the referee's integer chain predicate against oracle/exact.py's rational one, on lattice segments that touch, overlap
    and cross often"""
    from oracle import exact

    rng = np.random.default_rng(5)
    pts = [tuple(int(v) for v in rng.integers(0, 5, 2)) for _ in range(4 * 3000)]
    hits = 0
    for k in range(0, len(pts), 4):
        a0, a1, b0, b1 = pts[k:k + 4]
        want = exact.segments_intersect(a0, a1, b0, b1)
        assert R.segments_meet(a0, a1, b0, b1) == want, (a0, a1, b0, b1)
        hits += want
    assert 300 < hits < 2700


# ---- the oracle against the referee ------------------------------------------------------------------------------------
def column(kind, rows):
    return GeoArrowArray.from_shapes(T[kind], rows)


def grouped(cases):
    """{(kind_a, kind_b): (case indices, rows_a, rows_b)} of (kind_a, row_a, kind_b, row_b, ...) cases"""
    out = {}
    for i, c in enumerate(cases):
        g = out.setdefault((c[0], c[2]), ([], [], []))
        g[0].append(i), g[1].append(c[1]), g[2].append(c[3])
    return out


def referee(cases):
    """(intersects, true distance, ℓ) per case"""
    hit, true, ell = [], [], []
    for ka, a, kb, b, *_ in cases:
        hit.append(R.intersects(a, b, ka, kb))
        true.append(R.distance(a, b, ka, kb))
        ell.append(R.envelope_diagonal((ka, a), (kb, b)))
    return np.array(hit), true, np.array(ell)


def oracle_rowwise(og, conv, cases):
    inter = np.zeros(len(cases), bool)
    dist = np.zeros(len(cases))
    for (ka, kb), (idx, ra, rb) in grouped(cases).items():
        ga, gb = conv(column(ka, ra)), conv(column(kb, rb))
        inter[idx] = og.intersects_rowwise(ga, gb)
        dist[idx] = og.distance_rowwise(ga, gb)
    return inter, dist


def k_ratio(got, true, ell):
    """the K each row needs: |got − true| / (u (true + ℓ))"""
    err = [R.distance_error(g, t) for g, t in zip(got, true)]
    return np.array([x / (R.U * (float(t) + e)) if x else 0.0 for x, t, e in zip(err, true, ell)])


def checked_cases():
    a = []
    for ka in PF.KINDS:
        for kb in PF.KINDS:
            ra, rb = PF.family_a(ka, kb, 10)
            ox, oy = PF.A_OFFSETS[-1]
            a += [(ka, x, kb, y) for x, y in zip(ra, rb)]
            a += [(ka, PF.translate(x, ox, oy), kb, PF.translate(y, ox, oy)) for x, y in zip(ra, rb)]
    c = [r for r in PF.family_c() if len(r[1]) >= 2 and len(r[3]) >= 2]  # shorter rows: null distances, not in scope
    return {"A": a, "B": PF.family_b(), "C": c + PF.family_c_rings(), "D": PF.family_d()}


@pytest.fixture(scope="module")
def families():
    return checked_cases()


@pytest.mark.parametrize("fam", ["A", "B", "C", "D"])
def test_oracle_within_bound_of_referee(og, conv, families, fam):
    cases = families[fam]
    hit, true, ell = referee(cases)
    inter, dist = oracle_rowwise(og, conv, cases)
    assert np.array_equal(inter, hit)
    assert (dist[hit] == 0.0).all()
    k = k_ratio(dist, true, ell)
    print(f"family {fam}: {len(cases)} rows, {int(hit.sum())} intersecting, oracle max K = {k.max():.2f}")
    assert k.max() <= R.DISTANCE_K, np.argmax(k)
    assert hit.any() and not hit.all()


def test_oracle_contains_matches_referee(og, conv):
    n = 0
    for kind, a, p in PF.family_b_contains_point():
        got = og.contains_rowwise(conv(column(kind, [a])), np.array([p], float))[0]
        assert got == R.contains_point(kind, a, p), (kind, a, p)
        n += 1
    pos = 0
    for kind, a, b in PF.family_b_contains_polygon():
        got = og.contains_polygon_rowwise(conv(column(kind, [a])), conv(column("polygon", [b])))[0]
        want = R.contains_polygon(kind, a, b)
        assert got == want, (kind, a, b)
        pos += want
    assert n > 100 and 0 < pos


def test_oracle_bit_identical_under_exact_translation(og, conv):
    """family A: intersects and contains unchanged, distance bit for bit — geo's arithmetic works on coordinate differences"""
    rows = 0
    for ka in PF.KINDS:
        for kb in PF.KINDS:
            ra, rb = PF.family_a(ka, kb, 40)
            base_i = og.intersects_rowwise(conv(column(ka, ra)), conv(column(kb, rb)))
            base_d = og.distance_rowwise(conv(column(ka, ra)), conv(column(kb, rb)))
            assert base_i.any() and not base_i.all()
            for ox, oy in PF.A_OFFSETS[1:]:
                ta, tb = conv(column(ka, PF.translate(ra, ox, oy))), conv(column(kb, PF.translate(rb, ox, oy)))
                assert np.array_equal(og.intersects_rowwise(ta, tb), base_i)
                assert np.array_equal(og.distance_rowwise(ta, tb).view(np.uint64), base_d.view(np.uint64)), (ka, kb, ox, oy)
            rows += len(ra)
    A, B = PF.family_a_contains(40)
    base = og.contains_polygon_rowwise(conv(column("polygon", A)), conv(column("polygon", B)))
    for ox, oy in PF.A_OFFSETS[1:]:
        t = og.contains_polygon_rowwise(conv(column("polygon", PF.translate(A, ox, oy))), conv(column("polygon", PF.translate(B, ox, oy))))
        assert np.array_equal(t, base)
    assert base.any() and not base.all() and rows == 36 * 40
