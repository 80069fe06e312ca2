"""The row-wise `intersects`, `distance` and `contains` kernels against the exact referee tests/pairs_reference.py, on the
families of tests/pairs_families.py: far from the origin, at gaps of a few ulps, and at every row length where the LineString
kernels switch path (k_ls_ls_fast for <= 33 coordinates per side, the flagged exact redo, the long-row path).

Booleans must equal the referee's.  A distance must be 0 wherever the referee intersects and otherwise lie within
|got − true| <= K·u·(true + ℓ) (pairs_reference); a distance below K·u·ℓ may round to 0 (geo's epsilon-based point-on-line test
also returns 0 there, by design).  Each family prints the largest K any of its rows needs; on an H100 80GB HBM3 it was 0.44
(A), 0 (B: the gaps come out exact), 0.01 (C) and 0.80 (D), the CPU oracle's 0.55, 0, 0.02 and 0.80.  A relative tolerance (the 1e-9 of tests/test_gpu_predicates.py) cannot hold on family D:
a point 1e-12 from a segment between coordinates of 10⁷ carries an absolute error of order u·ℓ in any f64 evaluation."""
import numpy as np
import pytest

import pairs_families as PF
import pairs_reference as R
from geopolars_b200 import GeoArrowArray, GeometryType, engine

pytestmark = pytest.mark.gpu

T = {k: GeometryType[k.upper()] for k in PF.KINDS}


def column(kind, rows):
    return GeoArrowArray.from_shapes(T[kind], rows)


def gpu_rowwise(ctx, cases):
    """(intersects, distance, distance valid) of (kind_a, row_a, kind_b, row_b, ...) cases, one launch per type pair"""
    groups = {}
    for i, c in enumerate(cases):
        g = groups.setdefault((c[0], c[2]), ([], [], []))
        g[0].append(i), g[1].append(c[1]), g[2].append(c[3])
    inter, dist, valid = np.zeros(len(cases), bool), np.zeros(len(cases)), np.zeros(len(cases), bool)
    for (ka, kb), (idx, ra, rb) in groups.items():
        da, db = ctx.upload(column(ka, ra)), ctx.upload(column(kb, rb))
        inter[idx] = engine.intersects(da, db)
        dist[idx], valid[idx] = engine.distance(da, db)
    return inter, dist, valid


def check_against_referee(name, cases, inter, dist, valid):
    """booleans equal, 0 where the referee intersects, every distance within the bound; returns (rows, intersecting, max K)"""
    worst = 0.0
    hits = 0
    for i, (ka, a, kb, b, *_) in enumerate(cases):
        hit = R.intersects(a, b, ka, kb)
        assert inter[i] == hit, (name, i, ka, a, kb, b)
        assert valid[i], (name, i)
        true = R.distance(a, b, ka, kb)
        ell = R.envelope_diagonal((ka, a), (kb, b))
        if hit:
            assert dist[i] == 0.0, (name, i, dist[i])
            hits += 1
        err = R.distance_error(dist[i], true)
        assert err <= R.distance_bound(true, ell), (name, i, ka, a, kb, b, dist[i], float(true))
        if err:
            worst = max(worst, err / (R.U * (float(true) + ell)))
    print(f"family {name}: {len(cases)} rows checked against the referee, {hits} intersecting, max K = {worst:.2f}")
    return len(cases), hits, worst


# ---- A: exact translations --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ka", PF.KINDS)
def test_a_exact_translation_is_bit_identical(ctx, ka):
    """at every offset the translated columns give the origin's intersects, contains and join pairs, and bit for bit its
    distances (values and validity), areas and lengths; a subset is also checked against the referee"""
    n, rows = 300, 0
    for kb in PF.KINDS:
        ra, rb = PF.family_a(ka, kb, n)
        da, db = ctx.upload(column(ka, ra)), ctx.upload(column(kb, rb))
        base_i = engine.intersects(da, db)
        base_d, base_v = engine.distance(da, db)
        base_j = {p: engine.spatial_join(da, db, p) for p in ("intersects", "contains")}
        assert base_i.any() and not base_i.all() and base_v.all()
        pts = kb == "point" and ka not in ("point", "multipoint")
        base_c = engine.contains(da, db) if pts else None
        base_m = (engine.area(da), engine.euclidean_length(da)) if kb == "point" else None
        for ox, oy in PF.A_OFFSETS[1:]:
            ta, tb = ctx.upload(column(ka, PF.translate(ra, ox, oy))), ctx.upload(column(kb, PF.translate(rb, ox, oy)))
            assert np.array_equal(engine.intersects(ta, tb), base_i), (ka, kb, ox, oy)
            d, v = engine.distance(ta, tb)
            assert np.array_equal(v, base_v) and np.array_equal(d.view(np.uint64), base_d.view(np.uint64)), (ka, kb, ox, oy)
            for p, (l, r) in base_j.items():
                tl, tr = engine.spatial_join(ta, tb, p)
                assert np.array_equal(tl, l) and np.array_equal(tr, r), (ka, kb, p, ox, oy)
            if pts:
                assert np.array_equal(engine.contains(ta, tb), base_c)
            if base_m is not None:  # E: both work on differences from the ring's / line's first coordinate
                assert np.array_equal(engine.area(ta).view(np.uint64), base_m[0].view(np.uint64))
                assert np.array_equal(engine.euclidean_length(ta).view(np.uint64), base_m[1].view(np.uint64))
        rows += n * len(PF.A_OFFSETS)
        m = 12
        ox, oy = PF.A_OFFSETS[-1]
        sub = [(ka, x, kb, y) for x, y in zip(ra[:m], rb[:m])] + \
              [(ka, PF.translate(x, ox, oy), kb, PF.translate(y, ox, oy)) for x, y in zip(ra[:m], rb[:m])]
        check_against_referee(f"A {ka} x {kb}", sub, *gpu_rowwise(ctx, sub))
    print(f"family A, {ka} x every kind: {rows} rows compared with their origin copies")


def test_a_contains_polygon_translation(ctx):
    A, B = PF.family_a_contains(300)
    base = engine.contains(ctx.upload(column("polygon", A)), ctx.upload(column("polygon", B)))
    want = np.array([R.contains_polygon("polygon", a, b) for a, b in zip(A[:80], B[:80])])
    assert np.array_equal(base[:80], want) and base.any() and not base.all()
    for ox, oy in PF.A_OFFSETS[1:]:
        ga, gb = ctx.upload(column("polygon", PF.translate(A, ox, oy))), ctx.upload(column("polygon", PF.translate(B, ox, oy)))
        assert np.array_equal(engine.contains(ga, gb), base)
        assert all(np.array_equal(x, y) for x, y in zip(engine.spatial_join(ga, gb, "contains"),
                                                         engine.spatial_join(ctx.upload(column("polygon", A)), ctx.upload(column("polygon", B)), "contains")))


# ---- B: ulp gaps ------------------------------------------------------------------------------------------------------------
def test_b_ulp_gaps(ctx):
    cases = PF.family_b()
    inter, dist, valid = gpu_rowwise(ctx, cases)
    rows, hits, _ = check_against_referee("B", cases, inter, dist, valid)
    assert 0 < hits < rows
    # far from the origin a 1-ulp gap is far above the bound: those rows must be > 0, not rounded to "touching"
    far_gap = [i for i, c in enumerate(cases) if c[4] != 0.0 and not inter[i]]
    assert far_gap and (dist[far_gap] > 0.0).all()


def test_b_contains(ctx):
    n = hits = 0
    for kind, a, p in PF.family_b_contains_point():
        got = engine.contains(ctx.upload(column(kind, [a])), ctx.upload(GeoArrowArray.points(np.array([p], float))))[0]
        want = R.contains_point(kind, a, p)
        assert got == want, (kind, a, p)
        n, hits = n + 1, hits + want
    for kind, a, b in PF.family_b_contains_polygon():
        got = engine.contains(ctx.upload(column(kind, [a])), ctx.upload(column("polygon", [b])))[0]
        want = R.contains_polygon(kind, a, b)
        assert got == want, (kind, a, b)
        n, hits = n + 1, hits + want
    print(f"family B contains: {n} rows, {hits} contained")
    assert 0 < hits < n


# ---- C: lengths at the path switches ----------------------------------------------------------------------------------------
def test_c_linestring_lengths_in_one_launch(ctx, og, conv):
    """every (len_a, len_b) in C_LENGTHS² and every mode in ONE column, so short rows the fast path finishes, rows it flags
    (touching or 1 ulp apart: the filter cannot certify a sign) and long rows are all in the same launch"""
    rows = PF.family_c()
    ga, gb = column("linestring", [r[1] for r in rows]), column("linestring", [r[3] for r in rows])
    da, db = ctx.upload(ga), ctx.upload(gb)
    inter = engine.intersects(da, db)
    dist, valid = engine.distance(da, db)
    # rows with fewer than 2 coordinates on a side: geo panics in the distance (null), the oracle's NaN
    want_null = np.isnan(og.distance_rowwise(conv(ga), conv(gb)))
    assert np.array_equal(valid, ~want_null)
    assert np.array_equal(inter, og.intersects_rowwise(conv(ga), conv(gb)))
    short = [i for i, r in enumerate(rows) if len(r[1]) < 2 or len(r[3]) < 2]
    assert want_null[short].all() and not inter[short].any()
    keep = [i for i in range(len(rows)) if i not in set(short)]
    check_against_referee("C", [rows[i] for i in keep], inter[keep], dist[keep], valid[keep])
    modes = np.array([PF.C_MODES[i % len(PF.C_MODES)] for i in range(len(rows))])
    k = np.array(keep)
    assert inter[k][modes[k] == "touch"].all() and inter[k][modes[k] == "on_edge"].all()
    for m in ("ulp", "flat_ulp"):
        assert not inter[k][modes[k] == m].any() and (dist[k][modes[k] == m] > 0).all()


def test_c_rings_and_members_straddling_33(ctx):
    cases = PF.family_c_rings()
    rows, hits, _ = check_against_referee("C rings", cases, *gpu_rowwise(ctx, cases))
    assert 0 < hits < rows


# ---- D: badly conditioned distances -----------------------------------------------------------------------------------------
def test_d_badly_conditioned_distances(ctx):
    cases = PF.family_d()
    check_against_referee("D", cases, *gpu_rowwise(ctx, cases))
