"""Nearest join with a left side of any geometry type (gpl_nearest_join_geom*, DESIGN.md §4.13): every output is compared
bit for bit with a referee built from the row-wise `distance` entry point.  For a sampled left row the referee evaluates
`distance(lhs, rhs)` on a column of that row repeated once per right row (the left row first), drops the right rows
outside R and the pairs beyond max_distance or with a null distance, and takes the minimum, the lowest row at it and the
number of rows at it.  Left rows that are null, empty or have a non-finite coordinate match nothing."""
import math

import numpy as np
import pytest

import nearest_geom_reference as ngr
import nearest_reference as nr
import shapes
from geopolars_b200 import GeoArrowArray, GeometryType, _lib, engine
from geopolars_b200.geoseries import GeoSeries, nearest_join
from test_gpu_nearest import T, r_mask, same_f64

pytestmark = pytest.mark.gpu

INF = float("inf")
KINDS = list(T)


def to_og(a: GeoArrowArray):
    from oracle import oracle as og

    return og.OGArray(int(a.type), a.xy, geom_off=a.geom_off, part_off=a.part_off, ring_off=a.ring_off, valid=a.valid)


def repeat_row(a: GeoArrowArray, i: int, m: int) -> GeoArrowArray:
    if a.type == GeometryType.LINESTRING:  # direct, for right sides of millions of rows
        c = a.xy[a.geom_off[i]:a.geom_off[i + 1]]
        return GeoArrowArray.linestrings(np.tile(c, (m, 1)), np.arange(m + 1, dtype=np.int64) * len(c))
    t = nr.take(to_og(a), np.full(m, i, dtype=np.int64))
    return GeoArrowArray(a.type, t.xy, geom_off=t.geom_off, part_off=t.part_off, ring_off=t.ring_off)


def referee(ctx, lhs, rhs, rhs_dev, rows, maxd=INF):
    """(nearest_id, distance, n_tied, {k: tied rows}) for the left rows `rows`, by brute force through `distance`"""
    R = r_mask(rhs)
    L = r_mask(lhs)
    m = len(rhs)
    nid, dist, tied, out = [], [], [], {}
    for k, i in enumerate(rows):
        if not L[i] or m == 0:
            nid.append(-1), dist.append(np.nan), tied.append(0)
            continue
        d, valid = engine.distance(ctx.upload(repeat_row(lhs, i, m)), rhs_dev)
        ok = R & valid.astype(bool) & (d <= maxd)
        if not ok.any():
            nid.append(-1), dist.append(np.nan), tied.append(0)
            continue
        best = d[ok].min()
        js = np.nonzero(ok & (d == best))[0]
        nid.append(int(js[0])), dist.append(best), tied.append(len(js))
        out[k] = js
    return np.array(nid, np.int32), np.array(dist), np.array(tied, np.int32), out


def check_geom(ctx, lhs, rhs, maxd=INF, sample=None, idx=None, cpu=True):
    """join outputs for all left rows (+ pair list) == referee on `sample`; returns (idx, nid, dist, tied)"""
    rhs_dev = ctx.upload(rhs)
    idx = idx or engine.NearestIndex(rhs_dev)
    ld = ctx.upload(lhs)
    nid, dist, tied = idx.query_geom(ld, maxd)
    a, b, d2 = idx.pairs_geom(ld, maxd, with_distance=True)
    assert same_f64(d2, dist)
    sample = np.arange(len(lhs)) if sample is None else np.asarray(sample)
    rn, rd, rt, rows = referee(ctx, lhs, rhs, rhs_dev, sample, maxd)
    assert np.array_equal(nid[sample], rn), np.nonzero(nid[sample] != rn)[0][:10]
    assert same_f64(dist[sample], rd)
    assert np.array_equal(tied[sample], rt)
    # pair list: sorted, each tied row once, consistent with the dense form
    key = a.astype(np.int64) * (1 << 32) + b.astype(np.int64)
    assert np.all(np.diff(key) > 0)
    assert len(a) == int(tied.sum())
    starts = np.searchsorted(a, np.arange(len(lhs)))
    for k, i in enumerate(sample):
        got = b[starts[i]:starts[i] + tied[i]].astype(np.int64)
        assert np.array_equal(got, rows.get(k, np.zeros(0, np.int64))), i
    if cpu and len(rhs) * len(sample) <= 200_000:
        cn, cd, ct = ngr.nearest_join_geom(to_og(lhs), to_og(rhs), maxd, use_pruning=True)
        from conftest import rel_close

        assert np.array_equal(cn[sample] >= 0, nid[sample] >= 0)
        assert rel_close(cd[sample], dist[sample])
    return idx, nid, dist, tied


def rows_of(kind, rng, n, span=10.0):
    rows = shapes.random_rows(rng, kind, n, span) + ngr.planted(kind)
    return [rows[i] for i in rng.permutation(len(rows))]


@pytest.mark.parametrize("lk", [k for k in KINDS if k != "point"])
@pytest.mark.parametrize("rk", KINDS)
def test_every_type_pair_vs_referee(ctx, lk, rk):
    rng = np.random.default_rng(KINDS.index(lk) * 6 + KINDS.index(rk))
    rrows = rows_of(rk, rng, 120)
    lrows = shapes.random_rows(rng, lk, 50)
    if lk in ("multipoint", "linestring", "multilinestring"):  # left rows sharing a vertex or a segment point with a right row
        lrows = shapes.plant_touching(rng, lk, lrows, rk, rrows[:50], every=3)
    lrows = lrows + ngr.planted(lk)
    lrows = [lrows[i] for i in rng.permutation(len(lrows))]
    lhs = GeoArrowArray.from_shapes(T[lk], lrows)
    rhs = GeoArrowArray.from_shapes(T[rk], rrows)
    idx, nid, dist, tied = check_geom(ctx, lhs, rhs)
    assert idx.stats()["evaluations"] > 0
    L = r_mask(lhs)
    assert (nid[~L] == -1).all() and (tied[~L] == 0).all()


def test_point_left_side_equals_point_entries(ctx):
    rng = np.random.default_rng(1)
    for rk in KINDS:
        rhs = GeoArrowArray.from_shapes(T[rk], rows_of(rk, rng, 150))
        idx = engine.NearestIndex(ctx.upload(rhs))
        P = np.concatenate([rng.uniform(-2, 12, (200, 2)), [[np.nan, 1.0], [1e6, 0.0]]])
        pv = np.ones(len(P), bool)
        pv[::9] = False
        pd = ctx.upload(GeoArrowArray.points(P, valid=pv))
        for maxd in (INF, 0.5):
            g, p = idx.query_geom(pd, maxd), idx.query_array(pd, maxd)
            assert np.array_equal(g[0], p[0]) and same_f64(g[1], p[1]) and np.array_equal(g[2], p[2])
            ga, gb, gd = idx.pairs_geom(pd, maxd, with_distance=True)
            pa, pb, pdd = idx.pairs_array(pd, maxd, with_distance=True)
            assert np.array_equal(ga, pa) and np.array_equal(gb, pb) and same_f64(gd, pdd)


def test_ls_ls_fast_path_limit_and_uncertified_filter(ctx):
    """LineString x LineString on both sides of the 33-coordinate fast path, and collinear overlaps the fast filter
    cannot certify (they go to the exact routine, as in `distance`)"""
    rng = np.random.default_rng(2)

    def walk(n, x0, y0):
        p = np.array([x0, y0]) + np.cumsum(rng.uniform(-0.3, 0.3, (n, 2)), 0)
        return [tuple(q) for q in p]

    rrows = [walk(int(n), *rng.uniform(0, 20, 2)) for n in rng.choice([2, 5, 32, 33, 34, 40, 90], 300)]
    lrows = [walk(int(n), *rng.uniform(0, 20, 2)) for n in rng.choice([2, 33, 34, 70], 60)]
    # collinear and overlapping segments (uncertified signs), touching end points, a zero-length segment
    lrows += [[(1.0, 1.0), (3.0, 1.0)], [(2.0, 2.0), (2.0, 2.0), (5.0, 2.0)], [rrows[0][0], (50.0, 50.0)]]
    rrows += [[(0.0, 1.0), (2.0, 1.0), (4.0, 1.0)], [(3.0, 2.0), (4.0, 2.0)]]
    lhs = GeoArrowArray.from_shapes(GeometryType.LINESTRING, lrows)
    rhs = GeoArrowArray.from_shapes(GeometryType.LINESTRING, rrows)
    _, nid, dist, _ = check_geom(ctx, lhs, rhs)
    assert (dist[-3:] == 0.0).all()


def test_ls_ls_fraction_pick_is_kept(ctx):
    """single LineString x LineString pairs where gpl_distance's fast path (the minimum picked by cross-multiplied
    fractions) differs in the last ulp from sqrt(ls_ls_min_dist2), the value member_distance would give
    (tests/test_nearest_geom_bound_model.py finds them): the join must return gpl_distance's bits"""
    from test_nearest_geom_bound_model import fraction_cases, ls_ls_min, ls_ls_short

    cases = fraction_cases(3)
    assert len(cases) == 3
    lhs = GeoArrowArray.from_shapes(GeometryType.LINESTRING, [A for A, _ in cases])
    rhs = GeoArrowArray.from_shapes(GeometryType.LINESTRING, [B for _, B in cases])
    _, nid, dist, tied = check_geom(ctx, lhs, rhs, cpu=False)
    for i, (A, B) in enumerate(cases):
        d, _ = engine.distance(ctx.upload(GeoArrowArray.from_shapes(GeometryType.LINESTRING, [A])),
                               ctx.upload(GeoArrowArray.from_shapes(GeometryType.LINESTRING, [B])))
        assert d[0] == ls_ls_short(A, B) != ls_ls_min(A, B)  # the model of the fast path is the device's
        if nid[i] == i:
            assert dist[i] == d[0]
    # one pair per index: the nearest row is the planted one
    for A, B in cases:
        _, nid, dist, _ = check_geom(ctx, GeoArrowArray.from_shapes(GeometryType.LINESTRING, [A]),
                                     GeoArrowArray.from_shapes(GeometryType.LINESTRING, [B]), cpu=False)
        assert nid[0] == 0 and dist[0] == ls_ls_short(A, B) != ls_ls_min(A, B)


def test_invalid_polygons_and_hole_branch(ctx):
    """a hole outside the exterior, a hole containing the exterior (the representative-vertex bound would lose the true
    nearest row there), and left geometries inside valid holes (the hole branch of the distance runs)"""
    big_hole = [[(0.0, 0.0), (40.0, 0.0), (40.0, 40.0), (0.0, 40.0), (0.0, 0.0)], [(10.0, 10.0), (30.0, 10.0), (30.0, 30.0), (10.0, 30.0), (10.0, 10.0)]]
    hole_out = [[(50.0, 0.0), (51.0, 0.0), (51.0, 1.0), (50.0, 0.0)], [(60.0, 5.0), (61.0, 5.0), (61.0, 6.0), (60.0, 5.0)]]
    rpolys = [ngr.hole_contains_exterior(), big_hole, hole_out, [[(5.5, 0.2), (5.7, 0.2), (5.6, 0.4), (5.5, 0.2)]]]
    lsegs = [[(0.5, 0.5), (0.5, 0.6)], [(20.0, 20.0), (21.0, 21.0)], [(60.5, 5.2), (60.6, 5.3)], [(12.0, 12.0), (12.5, 13.0)]]
    lpolys = [[[(0.4, 0.4), (0.6, 0.4), (0.5, 0.6), (0.4, 0.4)]], [[(20.0, 20.0), (21.0, 20.0), (21.0, 21.0), (20.0, 20.0)]]]
    for rk, rrows in (("polygon", rpolys), ("multipolygon", [[p] for p in rpolys])):
        rhs = GeoArrowArray.from_shapes(T[rk], rrows)
        check_geom(ctx, GeoArrowArray.from_shapes(GeometryType.LINESTRING, lsegs), rhs)
        check_geom(ctx, GeoArrowArray.from_shapes(GeometryType.POLYGON, lpolys), rhs)
    # invalid polygons on the LEFT side, against lines and points
    rl = GeoArrowArray.from_shapes(GeometryType.LINESTRING, lsegs + [[(5.0, 0.5), (5.0, 0.6)]])
    check_geom(ctx, GeoArrowArray.from_shapes(GeometryType.POLYGON, rpolys), rl)
    rp = GeoArrowArray.points(np.array([[0.5, 0.5], [5.0, 0.5], [20.0, 20.0], [60.5, 5.5], [100.0, 0.0]]))
    check_geom(ctx, GeoArrowArray.from_shapes(GeometryType.POLYGON, rpolys), rp)
    # the U trap: a segment inside the exterior of the hole-contains-exterior polygon; its computed distance to that polygon
    # (~10.4, to the hole) exceeds that of a row at distance 5, which must be found
    rhs = GeoArrowArray.from_shapes(GeometryType.POLYGON, [ngr.hole_contains_exterior(), [[(5.5, 0.5), (6.0, 0.5), (6.0, 0.6), (5.5, 0.5)]]])
    _, nid, dist, _ = check_geom(ctx, GeoArrowArray.from_shapes(GeometryType.LINESTRING, [[(0.5, 0.5), (0.5, 0.6)]]), rhs)
    assert nid[0] == 1 and dist[0] == 5.0


def test_overlaps_touches_and_lattice_ties(ctx):
    sq = lambda x, y, s: [[(x, y), (x + s, y), (x + s, y + s), (x, y + s), (x, y)]]
    rhs = GeoArrowArray.from_shapes(GeometryType.POLYGON, [sq(float(x), float(y), 1.0) for x in range(20) for y in range(20)])
    # unit squares offset by half a cell: each touches / overlaps 4 lattice squares -> ties at 0
    lhs = GeoArrowArray.from_shapes(GeometryType.POLYGON, [sq(x + 0.5, y + 0.5, 0.25) for x in range(19) for y in range(19)] +
                                    [sq(x + 1.0, y + 1.0, 0.0) for x in range(3) for y in range(3)])
    _, nid, dist, tied = check_geom(ctx, lhs, rhs, sample=np.r_[0:40, 361:370])
    assert (dist == 0.0).all() and (tied[:361] == 1).all()
    # one square over the whole lattice: 400 rows tied at 0, more than the on-chip per-row sort takes
    _, nid, dist, tied = check_geom(ctx, GeoArrowArray.from_shapes(GeometryType.POLYGON, [sq(-1.0, -1.0, 22.0)]), rhs)
    assert nid[0] == 0 and dist[0] == 0.0 and tied[0] == 400
    # lattice of points, left segments centred between 4 of them: 4-way ties at equal f64 distances
    g = np.arange(25, dtype=np.float64)
    X, Y = np.meshgrid(g, g)
    pts = GeoArrowArray.points(np.stack([X.ravel(), Y.ravel()], 1))
    segs = GeoArrowArray.from_shapes(GeometryType.LINESTRING, [[(x + 0.5, y + 0.5), (x + 0.5, y + 0.5)] for x in range(24) for y in range(24)])
    _, nid, dist, tied = check_geom(ctx, segs, pts, sample=np.arange(0, 576, 7))
    assert (tied == 4).all() and (dist == dist[0]).all()


def test_max_distance(ctx):
    rng = np.random.default_rng(7)
    rhs = GeoArrowArray.from_shapes(GeometryType.POLYGON, shapes.random_rows(rng, "polygon", 150, span=100.0))
    lhs = GeoArrowArray.from_shapes(GeometryType.LINESTRING, shapes.random_rows(rng, "linestring", 60, span=120.0))
    idx = engine.NearestIndex(ctx.upload(rhs))
    ld = ctx.upload(lhs)
    _, d_all, _ = idx.query_geom(ld)
    k = int(np.nanargmax(d_all))
    dk = d_all[k]
    for maxd in (dk, np.nextafter(dk, 0.0), 0.0, INF, float(np.nanmedian(d_all))):
        check_geom(ctx, lhs, rhs, maxd=maxd, idx=idx, sample=np.r_[k, 0:20])
    n1, _, _ = idx.query_geom(ld, dk)
    n2, d2, _ = idx.query_geom(ld, np.nextafter(dk, 0.0))
    assert n1[k] >= 0 and n2[k] == -1 and np.isnan(d2[k])
    for bad in (math.nan, -1.0):
        with pytest.raises(_lib.GeopolarsError) as e:
            idx.query_geom(ld, bad)
        assert e.value.code == -7
        with pytest.raises(_lib.GeopolarsError):
            idx.pairs_geom(ld, bad)


def test_regimes(ctx):
    """left boxes spanning the whole grid, 1e6 outside it, zero-width / zero-height right boxes"""
    rng = np.random.default_rng(5)
    rhs = GeoArrowArray.from_shapes(GeometryType.LINESTRING, shapes.random_rows(rng, "linestring", 400, span=100.0))
    lhs = GeoArrowArray.from_shapes(GeometryType.LINESTRING, [[(-50.0, -50.0), (150.0, 150.0)], [(-50.0, 60.0), (150.0, 61.0)],
                                                              [(1e6, 5.0), (1e6 + 1.0, 6.0)], [(-1e6, -1e6), (-1e6, 1e6)],
                                                              [(5e5, 5e5), (5e5, 5e5 + 1.0)]])
    check_geom(ctx, lhs, rhs)
    flat = GeoArrowArray.from_shapes(GeometryType.LINESTRING, [[(x, 0.0), (x + 0.5, 0.0)] for x in np.sort(rng.uniform(0, 100, 500))])
    tall = GeoArrowArray.points(np.stack([np.full(300, 2.5), rng.uniform(0, 10, 300)], 1))
    left = GeoArrowArray.from_shapes(GeometryType.POLYGON, shapes.random_rows(rng, "polygon", 40, span=100.0) +
                                     [[[(-10.0, -10.0), (110.0, -10.0), (110.0, 10.0), (-10.0, -10.0)]]])
    check_geom(ctx, left, flat)
    check_geom(ctx, left, tall)


def test_grid_cap(ctx):
    """>= 4.2 M right rows: the index reaches the 2048-cell cap; left lines, polygons and far-away rows against it"""
    import torch

    n = 4_300_000
    xy = torch.empty((n, 2), dtype=torch.float64, device="cuda")
    engine.check(ctx.lib.gpl_gen_uniform_points(ctx._h, 9, 0, n, 1000.0, xy.data_ptr()))
    ctx.synchronize()
    host = xy.cpu().numpy()
    rhs = GeoArrowArray.points(host)
    rhs_dev = ctx.upload(rhs)
    idx = engine.NearestIndex(rhs_dev)
    assert idx.stats()["grid_cells_per_axis"] == 2048
    rng = np.random.default_rng(2)
    rows = [[tuple(p), tuple(p + rng.uniform(-0.2, 0.2, 2))] for p in rng.uniform(-10, 1010, (10, 2))]
    rows += [[tuple(host[0] + 1e-9), tuple(host[0] + 0.01)], [(5e5, 5e5), (5e5 + 1.0, 5e5)], [(0.0, 500.0), (1000.0, 500.5)]]
    lhs = GeoArrowArray.from_shapes(GeometryType.LINESTRING, rows)
    ld = ctx.upload(lhs)
    nid, dist, tied = idx.query_geom(ld)
    a, b, d2 = idx.pairs_geom(ld, with_distance=True)
    assert same_f64(d2, dist) and len(a) == int(tied.sum())
    rn, rd, rt, out = referee(ctx, lhs, rhs, rhs_dev, np.arange(len(rows)))
    assert np.array_equal(nid, rn) and same_f64(dist, rd) and np.array_equal(tied, rt)
    starts = np.searchsorted(a, np.arange(len(rows)))
    for k in range(len(rows)):
        assert np.array_equal(b[starts[k]:starts[k] + tied[k]].astype(np.int64), out.get(k, np.zeros(0, np.int64)))
    assert idx.stats()["evaluations"] < 2_000_000  # pruned: the grid, not a scan of 4.3 M rows per left row (13 rows)


def test_slack_keeps_rows_computed_below_their_box_distance(ctx):
    """the case the bound model's tau = 0 control finds (tests/test_nearest_geom_bound_model.py): a left segment whose
    computed LineString x LineString distance to a long segment is below their box distance, a parallel segment one ulp
    farther, and enough filler rows that the long segment lies one ring out.  Only the slack keeps the true nearest row."""
    from test_nearest_geom_bound_model import slack_cases

    for p, L, dB, fill in slack_cases(2):
        rows = [[(0.0, 0.0), (L, 0.0)], [(p[0] - dB, p[1]), (p[0] - dB, p[1] + 1.0)]] + fill
        rhs = GeoArrowArray.from_shapes(GeometryType.LINESTRING, rows)
        lhs = GeoArrowArray.from_shapes(GeometryType.LINESTRING, [[p, (p[0], p[1] + 1.0)]])
        _, nid, dist, tied = check_geom(ctx, lhs, rhs, cpu=False)
        assert nid[0] == 0 and tied[0] == 1 and dist[0] < p[1]


def test_queue_drains_and_continues(ctx):
    """a left polygon overlapping 3 000 right rows (and a few of the scattered ones): they all tie at 0, many times the
    per-warp queue"""
    rng = np.random.default_rng(11)
    rows = [[shapes.star_ring(rng, *rng.uniform(40, 60, 2), 5.0, 6, q=3)] for _ in range(3000)]
    rows += [[shapes.star_ring(rng, *rng.uniform(-100, 200, 2), 2.0, 6, q=3)] for _ in range(300)]
    rhs = GeoArrowArray.from_shapes(GeometryType.POLYGON, rows)
    lhs = GeoArrowArray.from_shapes(GeometryType.POLYGON, [[[(30.0, 30.0), (70.0, 30.0), (70.0, 70.0), (30.0, 70.0), (30.0, 30.0)]],
                                                           [[(-100.0, -100.0), (200.0, -100.0), (200.0, 200.0), (-100.0, -100.0)]]])
    idx, nid, dist, tied = check_geom(ctx, lhs, rhs, cpu=False)
    assert tied[0] >= 3000 and dist[0] == 0.0
    assert idx.stats()["evaluations"] >= 3000


def test_everywhere_rows_on_both_sides(ctx):
    """right rows with an empty member are evaluated for every left row; irregular left rows against every right row"""
    sq = lambda x, y: [(x, y), (x + 1, y), (x + 1, y + 1), (x, y + 1), (x, y)]
    rng = np.random.default_rng(3)
    rrows = [[[sq(x, y)]] for x, y in rng.uniform(0, 50, (300, 2))] + [[[sq(80.0, 80.0)], []]]
    rhs = GeoArrowArray.from_shapes(GeometryType.MULTIPOLYGON, rrows)
    lrows = [[[(x, y), (x + 0.2, y + 0.1)]] for x, y in rng.uniform(0, 50, (40, 2))] + [[[(3.0, 3.0)], [(9.0, 9.0), (9.5, 9.0)]], [[], [(1.0, 1.0), (2.0, 2.0)]]]
    lhs = GeoArrowArray.from_shapes(GeometryType.MULTILINESTRING, lrows)
    idx, nid, dist, tied = check_geom(ctx, lhs, rhs)
    assert idx.stats()["everywhere"] == 1
    # against a line side the empty member makes that row's distance null; against a MultiPoint side a 1-coordinate right
    # linestring is a real answer: geo's point rule gives 0 within 1.19e-7 of its coordinate (and f64::MAX beyond it), and
    # only the everywhere list reaches it
    rl = GeoArrowArray.from_shapes(GeometryType.LINESTRING, [[(float(x), float(y)), (x + 0.5, y + 0.5)] for x, y in rng.uniform(0, 50, (200, 2))] +
                                   [[(20.0, 20.0)], [(70.0, 70.0)]])
    lm = GeoArrowArray.from_shapes(GeometryType.MULTIPOINT, [[(20.0 + 1e-7, 20.0)], [(70.0, 70.0 - 5e-8), (60.0, 60.0)], [(100.0, 100.0)],
                                                              [(25.0, 25.0), (20.0, 20.0)]])
    idx, nid, dist, tied = check_geom(ctx, lm, rl)
    assert idx.stats()["everywhere"] == 2
    assert nid[0] == 200 and nid[1] == 201 and nid[3] == 200 and dist[0] == dist[1] == dist[3] == 0.0


def test_bundled_datasets(ctx):
    from geopolars_b200 import datasets

    cities = datasets.read_dataset("naturalearth_cities").geometry.device.to_host()
    countries = datasets.read_dataset("naturalearth_lowres").geometry.device.to_host()
    nybb = datasets.read_dataset("nybb").geometry.device.to_host()
    rng = np.random.default_rng(4)
    check_geom(ctx, countries, countries, sample=rng.choice(len(countries), 25, replace=False), cpu=False)
    check_geom(ctx, nybb, nybb, cpu=False)
    check_geom(ctx, countries, cities, sample=rng.choice(len(countries), 40, replace=False), cpu=False)


def test_million_walks_config2(ctx):
    """1 M 16-vertex walk linestrings x config 2's 10 k polygons; 2 000 left rows against the referee"""
    import torch

    from geopolars_b200 import synth

    m, grid, cell, nv = 10_000, 100, 10.0, 64
    pxy, ro, go = synth.star_polygons(m, grid, cell, nv)
    polys = GeoArrowArray.polygons(pxy, ro, go)
    n, k = 1_000_000, 16
    xy = torch.empty((n * k, 2), dtype=torch.float64, device="cuda")
    off = torch.empty(n + 1, dtype=torch.int64, device="cuda")
    engine.check(ctx.lib.gpl_gen_walk_linestrings(ctx._h, 3, -1, 0, n, k, xy.data_ptr(), off.data_ptr()))
    ctx.synchronize()
    walks = GeoArrowArray.linestrings(xy.cpu().numpy(), off.cpu().numpy())
    rhs_dev = ctx.upload(polys)
    idx = engine.NearestIndex(rhs_dev)
    ld = ctx.upload(walks)
    nid, dist, tied = idx.query_geom(ld)
    assert (nid >= 0).all() and (tied >= 1).all()
    s = np.random.default_rng(8).choice(n, 2000, replace=False)
    rn, rd, rt, _ = referee(ctx, walks, polys, rhs_dev, s)
    assert np.array_equal(nid[s], rn) and same_f64(dist[s], rd) and np.array_equal(tied[s], rt)


def test_nearest_join_any_left_type(ctx):
    rng = np.random.default_rng(9)
    rhs = GeoArrowArray.from_shapes(GeometryType.POLYGON, shapes.random_rows(rng, "polygon", 100))
    lrows = shapes.random_rows(rng, "linestring", 60, span=14.0) + [None, [], [(np.nan, 1.0), (2.0, 2.0)]]
    lhs_h = GeoArrowArray.from_shapes(GeometryType.LINESTRING, lrows)
    lhs = GeoSeries(_device=ctx.upload(lhs_h))
    rs = GeoSeries(_device=ctx.upload(rhs))
    idx = engine.NearestIndex(rs.device)
    a, b, d = nearest_join(lhs, rs)
    nid, dist, tied = idx.query_geom(lhs.device)
    la, lb = idx.pairs_geom(lhs.device)
    assert np.array_equal(a, la) and np.array_equal(b, lb) and same_f64(d, dist[a])
    assert not np.isin([60, 61, 62], a).any()
    a2, b2, d2 = nearest_join(lhs, rs, how="left", max_distance=0.5)
    _, _, tied2 = idx.query_geom(lhs.device, 0.5)
    miss = np.nonzero(tied2 == 0)[0]
    assert {60, 61, 62} <= set(miss.tolist())
    assert len(a2) == int(tied2.sum()) + len(miss) and sorted(set(a2.tolist())) == list(range(len(lrows)))
    assert (b2[np.isin(a2, miss)] == -1).all() and np.isnan(d2[np.isin(a2, miss)]).all()


def test_left_row_guard(ctx):
    """more than 2^31 - 1 left rows: GPL_ERR_UNSUPPORTED before any access (the column's buffers are never touched)"""
    import ctypes as C

    rhs = GeoArrowArray.from_shapes(GeometryType.POLYGON, [shapes.random_polygon(np.random.default_rng(0))])
    idx = engine.NearestIndex(ctx.upload(rhs))
    import torch

    small = torch.zeros(16, dtype=torch.int64, device="cuda")  # stands in for buffers of 2^31 rows: never read
    big = ctx.wrap_device(GeometryType.LINESTRING, 1 << 31, 1 << 32, small.data_ptr(), geom_off_ptr=small.data_ptr(), keepalive=(small,))
    buf = np.zeros(8, np.int32)
    rc = ctx.lib.gpl_nearest_join_geom(ctx._h, idx._h, big._h, math.nan, C.c_void_p(buf.ctypes.data), None, None, engine.GPL_DEVICE)
    assert rc == -6
    h = C.c_void_p()
    rc = ctx.lib.gpl_nearest_join_geom_pairs(ctx._h, idx._h, big._h, math.inf, C.byref(h), None, engine.GPL_DEVICE)
    assert rc == -6
    # the existing Point entry points still reject a non-Point left side
    with pytest.raises(_lib.MismatchedGeometry):
        idx.query_array(ctx.upload(rhs))
