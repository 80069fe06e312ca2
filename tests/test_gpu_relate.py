"""gpl_relate, the named DE-9IM predicates and the predicate join on the GPU (DESIGN.md §4.20).

  - against the exact referee tests/relate_reference.py, entry for entry: the hand cases, every one of the 36 type pairs of
    family A (planted shared vertices and vertices on edges), translated far from the origin by A_OFFSETS, the ulp-gap cases
    of family B, and rings / members of 31 to 35 coordinates and longer (family C rings, 64-vertex stars);
  - against the existing kernels at scale: "not disjoint" is bit-identical to `intersects` on every type pair, the DE-9IM
    contains to `contains` wherever that is defined;
  - analytic truth on lattices of unit squares;
  - the join against brute-force row-wise predicates over all pairs, and the points-in-polygons route against the relate route;
  - nulls, empty and non-finite rows, a length mismatch, a bad pattern and `disjoint` in the join."""
import numpy as np
import pytest

import pairs_families as PF
import relate_reference as R
import shapes
from geopolars_b200 import GeoArrowArray, GeometryType, engine as E
from geopolars_b200 import geoseries as gs

pytestmark = pytest.mark.gpu

T = {k: GeometryType[k.upper()] for k in PF.KINDS}
PREDICATES = ["intersects", "contains", "within", "contains_properly", "covers", "covered_by", "touches", "crosses", "overlaps",
              "geom_equals"]


def col(ctx, kind, rows):
    return ctx.upload(GeoArrowArray.from_shapes(T[kind], rows))


def mstr(m):
    return "".join("F" if v < 0 else str(v) for v in m)


def gpu_matrices(ctx, cases):
    """the matrix strings of (kind_a, row_a, kind_b, row_b, ...) cases, one launch per type pair"""
    groups = {}
    for i, c in enumerate(cases):
        g = groups.setdefault((c[0], c[2]), ([], [], []))
        g[0].append(i), g[1].append(c[1]), g[2].append(c[3])
    out = [None] * len(cases)
    for (ka, kb), (idx, ra, rb) in groups.items():
        m, valid = E.relate(col(ctx, ka, ra), col(ctx, kb, rb))
        assert valid.all()
        for i, row in zip(idx, m):
            out[i] = mstr(row)
    return out


def check_cases(ctx, cases):
    got = gpu_matrices(ctx, cases)
    for c, g in zip(cases, got):
        assert g == R.relate(c[0], c[1], c[2], c[3]), c


def sq(x, y, s):
    return [(x, y), (x + s, y), (x + s, y + s), (x, y + s), (x, y)]


def test_hand_cases(ctx):
    import test_relate_reference_cpu as H

    got = gpu_matrices(ctx, H.HAND)
    assert got == [c[4] for c in H.HAND]


@pytest.mark.parametrize("ka", PF.KINDS)
def test_family_a_against_referee(ctx, ka):
    cases = []
    for kb in PF.KINDS:
        ra, rb = PF.family_a(ka, kb, 24)
        cases += [(ka, a, kb, b) for a, b in zip(ra, rb)]
    check_cases(ctx, cases)
    # far from the origin: the translated rows give the origin's matrices (every coordinate difference is exact)
    want = gpu_matrices(ctx, cases)
    for ox, oy in PF.A_OFFSETS[1:]:
        moved = [(c[0], PF.translate(c[1], ox, oy), c[2], PF.translate(c[3], ox, oy)) for c in cases]
        assert gpu_matrices(ctx, moved) == want, (ox, oy)


def test_family_b_ulp_gaps(ctx):
    check_cases(ctx, [c[:4] for c in PF.family_b()])


def test_long_rows(ctx):
    cases = [c for c in PF.family_c_rings()]
    rng = np.random.default_rng(7)
    for k in range(12):
        a = shapes.valid_star(rng, 5, 5, 4.0, 64, q=3)
        b = shapes.valid_star(rng, 5 + 0.5 * (k % 3), 5, 3.0, 33 + k, q=3)
        cases += [("polygon", [a], "polygon", [b]), ("polygon", [a], "linestring", b), ("linestring", a[:40], "polygon", [b])]
    check_cases(ctx, cases)


@pytest.mark.parametrize("ka", PF.KINDS)
def test_against_existing_kernels_at_scale(ctx, ka):
    rng = np.random.default_rng(11)
    for kb in PF.KINDS:
        ra = shapes.random_rows(rng, ka, 20000)
        rb = shapes.random_rows(rng, kb, 20000)
        da, db = col(ctx, ka, ra), col(ctx, kb, rb)
        ok = (E.is_valid(da)[0] == 0) & (E.is_valid(db)[0] == 0)  # relate is defined for valid rows
        assert ok.mean() > 0.5
        inter = E.intersects(da, db)
        assert (~E.relate_predicate(da, db, "disjoint") == inter)[ok].all(), (ka, kb)
        assert (E.relate_predicate(da, db, "intersects") == inter)[ok].all(), (ka, kb)
        if (kb == "point" and R.CLASS[ka] >= 1) or (kb == "polygon" and R.CLASS[ka] == 2):
            got = E.relate_predicate(da, db, "contains")
            assert (got[ok] == E.contains(da, db)[ok]).all(), (ka, kb)


def _pairs(a, b):
    return sorted(zip(a.tolist(), b.tolist()))


def test_lattice(ctx):
    n = 24
    unit = [[sq(i, j, 1)] for j in range(n) for i in range(n)]
    du = col(ctx, "polygon", unit)
    cheb = {(p, q) for p in range(n * n) for q in range(n * n) if max(abs(p % n - q % n), abs(p // n - q // n)) == 1}
    assert set(_pairs(*E.predicate_join(du, du, "touches"))) == cheb
    assert _pairs(*E.predicate_join(du, du, "geom_equals")) == [(p, p) for p in range(n * n)]
    assert set(_pairs(*E.predicate_join(du, du, "intersects"))) == cheb | {(p, p) for p in range(n * n)}
    big = [[sq(2 * i, 2 * j, 2)] for j in range(n // 2) for i in range(n // 2)]
    db = col(ctx, "polygon", big)
    owner = [(p, (p // n // 2) * (n // 2) + (p % n) // 2) for p in range(n * n)]
    assert _pairs(*E.predicate_join(du, db, "within")) == owner
    assert _pairs(*E.predicate_join(du, db, "covered_by")) == owner
    assert _pairs(*E.predicate_join(db, du, "covers")) == sorted((q, p) for p, q in owner)
    assert len(E.predicate_join(db, du, "contains_properly")[0]) == 0  # every unit cell shares its big cell's boundary
    assert len(E.predicate_join(db, du, "contains")[0]) == n * n


@pytest.mark.parametrize("kinds", [("polygon", "linestring"), ("multipolygon", "polygon")])
def test_join_against_brute_force(ctx, kinds):
    ka, kb = kinds
    ra, _ = PF.family_a(ka, "point", 200)
    rb, _ = PF.family_a(kb, "point", 150)
    ra, rb = ra + [None], rb + [None]
    nl, nr = len(ra), len(rb)
    da, db = col(ctx, ka, ra), col(ctx, kb, rb)
    rep_a = col(ctx, ka, [ra[i] for i in range(nl) for _ in range(nr)])
    rep_b = col(ctx, kb, [rb[j] for _ in range(nl) for j in range(nr)])
    ga, gb = gs.GeoSeries(_device=da), gs.GeoSeries(_device=db)
    for pred in PREDICATES + ["relate_pattern"]:
        pat = "T*T***T**" if pred == "relate_pattern" else None
        bits = E.relate_predicate(rep_a, rep_b, pred, pat).reshape(nl, nr)
        want_l, want_r = np.nonzero(bits)
        a, b = E.predicate_join(da, db, pred, pat)
        assert a.tolist() == want_l.tolist() and b.tolist() == want_r.tolist(), pred
        a, b = gs.predicate_join(ga, gb, pred, how="left", pattern=pat)
        miss = [i for i in range(nl) if not bits[i].any()]
        wl = np.concatenate([want_l, miss]).astype(np.int64)
        wr = np.concatenate([want_r, np.full(len(miss), -1)]).astype(np.int64)
        order = np.lexsort((wr, wl))
        assert a.tolist() == wl[order].tolist() and b.tolist() == wr[order].tolist(), pred


def test_points_in_polygons_route(ctx):
    rng = np.random.default_rng(5)
    polys = [[shapes.valid_star(rng, float(rng.uniform(0, 100)), float(rng.uniform(0, 100)), 0.6, 8, q=3)] for _ in range(10_000)]
    dp = col(ctx, "polygon", polys)
    xy = np.round(rng.uniform(0, 100, (1_000_000, 2)), 3)
    xy[:1000] = np.array([p[0][0] for p in polys[:1000]])  # polygon vertices: on the boundary, never within
    pts = ctx.upload_separated(GeometryType.POINT, xy[:, 0], xy[:, 1])
    gp, gpoly = gs.GeoSeries(_device=pts), gs.GeoSeries(_device=dp)
    a, b = gs.predicate_join(gp, gpoly, "within")  # the points-in-polygons index
    ra, rb = E.predicate_join(pts, dp, "within")  # the DE-9IM route
    assert len(a) > 100_000
    assert a.tolist() == ra.astype(np.int64).tolist() and b.tolist() == rb.astype(np.int64).tolist()
    a, b = gs.predicate_join(gpoly, gp, "contains")
    ra, rb = E.predicate_join(dp, pts, "contains")
    assert a.tolist() == ra.astype(np.int64).tolist() and b.tolist() == rb.astype(np.int64).tolist()


def test_edge_cases(ctx):
    A = [[sq(0, 0, 2)], None, [], [sq(0, 0, 2)], [[(0, 0), (np.nan, 0), (1, 1), (0, 0)]], []]
    B = [[sq(1, 1, 2)], [sq(0, 0, 1)], [sq(0, 0, 1)], None, [sq(0, 0, 1)], []]
    da, db = col(ctx, "polygon", A), col(ctx, "polygon", B)
    m, valid = E.relate(da, db)
    assert valid.tolist() == [True, False, True, False, False, True]
    assert mstr(m[0]) == "212101212" and mstr(m[2]) == "FFFFFF212" and mstr(m[5]) == "FFFFFFFF2"
    s = gs.GeoSeries(_device=da).geo.relate(gs.GeoSeries(_device=db)).to_pylist()
    assert s == ["212101212", None, "FFFFFF212", None, None, "FFFFFFFF2"]
    assert E.relate_predicate(da, db, "intersects").tolist() == [True, False, False, False, False, False]
    assert E.relate_predicate(da, db, "geom_equals").tolist() == [False, False, False, False, False, True]
    assert E.relate_predicate(da, db, "relate_pattern", "2*t***t**").tolist() == [True] + [False] * 5
    with pytest.raises(ValueError):
        E.relate_predicate(da, db, "relate_pattern", "T*T***T*")
    with pytest.raises(ValueError):
        E.relate_predicate(da, db, "relate_pattern", "T*T***T*X")
    with pytest.raises(ValueError):
        E.predicate_join(da, db, "disjoint")
    with pytest.raises(ValueError):
        E.predicate_join(da, db, "relate_pattern", "FF*FF****")
    with pytest.raises(ValueError):
        E.relate(da, col(ctx, "polygon", A[:2]))
    # touches is false for two point columns whatever the matrix
    p = col(ctx, "point", [(0, 0), (1, 1)])
    assert E.relate_predicate(p, p, "touches").tolist() == [False, False]
    assert E.relate_predicate(p, p, "geom_equals").tolist() == [True, True]
