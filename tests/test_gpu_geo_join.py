"""Great-circle distance and joins for (lon, lat) degree Point columns (gpl_haversine_distance, gpl_geo_*, DESIGN.md §4.15).
Every join output is compared bit for bit with a referee built from the row-wise `haversine_distance` entry point: the left
row repeated once per right row, the eligibility mask, then `d <= D` or minimum / lowest row / ties.  Where sizes allow the
CPU reference (tests/geo_join_reference.py: cKDTree on unit vectors + the oracle's haversine) is compared too."""
import math

import numpy as np
import pytest

import geo_join_reference as gref
from geopolars_b200 import GeoArrowArray, GeometryType, _lib, engine
from geopolars_b200.geoseries import GeoSeries, geo_dwithin_join, geo_nearest_join

pytestmark = pytest.mark.gpu

R = 6371008.8
HALF = math.pi * R
INF = math.inf


def same_f64(a, b):
    return np.array_equal(np.asarray(a, np.float64).view(np.int64), np.asarray(b, np.float64).view(np.int64))


def sphere(rng, n, lon0=-180.0, lon1=180.0):
    return np.column_stack([rng.uniform(lon0, lon1, n), np.degrees(np.arcsin(rng.uniform(-1, 1, n)))])


def referee(ctx, p, Rr, rhs_dev, re):
    """distances of left point p to every right row through gpl_haversine_distance; NaN where the row is ineligible"""
    d, valid = engine.haversine_distance(ctx.upload(GeoArrowArray.points(np.repeat(p[None, :], len(Rr), axis=0))), rhs_dev)
    return np.where(re & valid.astype(bool), d, np.nan)


def check(ctx, L, Rr, D=None, maxd=INF, lvalid=None, rvalid=None, sample=None, cpu=True):
    """dwithin (when D is given) and nearest outputs == referee on `sample`; pair lists sorted and consistent with the dense
    outputs; the two joins consistent with each other.  Returns the index."""
    L, Rr = np.asarray(L, np.float64).reshape(-1, 2), np.asarray(Rr, np.float64).reshape(-1, 2)
    rhs_dev = ctx.upload(GeoArrowArray.points(Rr, valid=rvalid))
    ld = ctx.upload(GeoArrowArray.points(L, valid=lvalid))
    idx = engine.GeoIndex(rhs_dev)
    le, re = gref.eligible(L, lvalid), gref.eligible(Rr, rvalid)
    st = idx.stats()
    assert st["rows"] == int(re.sum()) and st["ineligible"] == int((~re).sum()) and st["cell_items"] == st["rows"]
    sample = np.arange(len(L)) if sample is None else np.asarray(sample)
    ref = {int(i): referee(ctx, L[i], Rr, rhs_dev, re) if le[i] and len(Rr) else np.full(len(Rr), np.nan) for i in sample}
    nid, dist, tied = idx.query(ld, None if maxd == INF else maxd)
    a, b, dd = idx.pairs(ld, None if maxd == INF else maxd, with_distance=True)
    assert same_f64(dd, dist) and np.all(np.diff(a.astype(np.int64) * (1 << 32) + b.astype(np.int64)) > 0)
    assert np.array_equal(np.bincount(a.astype(np.int64), minlength=len(L)), tied)
    assert np.array_equal(nid >= 0, tied > 0) and np.array_equal(nid < 0, np.isnan(dist))
    ts = np.concatenate([[0], np.cumsum(tied.astype(np.int64))])
    for i, d in ref.items():
        ok = ~np.isnan(d)
        u = d[ok].min() if ok.any() else np.nan
        if not ok.any() or not u <= maxd:
            assert nid[i] == -1 and tied[i] == 0, i
            continue
        want = np.nonzero(d == u)[0]
        assert nid[i] == want[0] and same_f64(dist[i], u) and np.array_equal(b[ts[i]:ts[i + 1]].astype(np.int64), want), i
    if D is not None:
        cnt = idx.count_within(ld, D)
        assert st["rows"] == 0 or len(L) == 0 or not le.any() or idx.stats()["evaluations"] >= int(cnt.sum())
        wa, wb, wd = idx.pairs_within(ld, D, with_distance=True)
        assert np.all(np.diff(wa.astype(np.int64) * (1 << 32) + wb.astype(np.int64)) > 0)
        assert np.array_equal(np.bincount(wa.astype(np.int64), minlength=len(L)), cnt)
        ws = np.concatenate([[0], np.cumsum(cnt.astype(np.int64))])
        for i, d in ref.items():
            js = np.nonzero(d <= D)[0]
            assert np.array_equal(wb[ws[i]:ws[i + 1]].astype(np.int64), js) and same_f64(wd[ws[i]:ws[i + 1]], d[js]), i
        # the two joins agree: the nearest distance is the minimum of the row's dwithin distances, its ties are among them
        near_D = idx.query(ld, D)
        assert np.array_equal(near_D[0] >= 0, cnt > 0)
        has = np.nonzero(cnt > 0)[0]
        assert same_f64(near_D[1][has], np.minimum.reduceat(wd, ws[has])) if len(has) else True
        key = set(zip(wa.tolist(), wb.tolist()))
        pa, pb = idx.pairs(ld, D)
        assert all((x, y) in key for x, y in zip(pa.tolist(), pb.tolist()))
    if cpu and len(Rr) * len(sample) <= 400_000:
        cn, cd, _ = gref.nearest(L[sample], Rr, maxd, None if lvalid is None else lvalid[sample], rvalid)
        gd = dist[sample]
        assert np.array_equal(np.isnan(cd), np.isnan(gd)) or maxd != INF
        both = ~np.isnan(cd) & ~np.isnan(gd)
        assert np.all(np.abs(cd[both] - gd[both]) <= 1e-9 * np.maximum(cd[both], 1.0))
    return idx


def fixture(rng, n, m):
    def cluster(c, k, s):
        return np.column_stack([c[0] + rng.uniform(-s, s, k), np.clip(c[1] + rng.uniform(-s, s, k), -90, 90)])

    Rr = np.concatenate([sphere(rng, m), cluster((179.9, 10.0), 30, 0.3), cluster((180.2, 10.0), 30, 0.3), cluster((0.0, 89.8), 20, 0.2),
                         cluster((50.0, -89.9), 20, 0.1), [[10.0, 20.0], [10.0, 20.0], [12.0, 20.0], [8.0, 20.0], [0.0, 90.0], [77.0, 90.0]],
                         [[np.nan, np.nan], [np.inf, 0.0], [0.0, 90.5], [360.5, 0.0], [5.0, np.nan]]])
    L = np.concatenate([sphere(rng, n, -180.0, 360.0),
                        [[180.0, 10.0], [-180.0, 10.0], [179.99, 10.1], [10.0, 20.0], [10.0, 25.0], [0.0, 90.0], [33.0, -90.0], [np.nan, np.nan],
                         [0.0, -91.0], [-360.5, 3.0], [np.inf, 3.0]]])
    lv, rv = np.ones(len(L), bool), np.ones(len(Rr), bool)
    lv[::11] = False
    rv[::13] = False
    return L, lv, Rr, rv


def test_haversine_distance_rowwise(ctx, og):
    rng = np.random.default_rng(1)
    P = np.concatenate([sphere(rng, 3000, -360, 360), [[0, 0], [0, 0], [179.9, 0], [0, 90], [np.nan, np.nan], [1, 2], [np.inf, 0], [5, np.nan]]])
    Q = np.concatenate([sphere(rng, 3000, -360, 360), [[90, 0], [180, 0], [-179.9, 0], [0, -90], [1, 2], [np.nan, np.nan], [0, 0], [5, 5]]])
    pv = np.ones(len(P), bool)
    pv[::17] = False
    a, b = ctx.upload(GeoArrowArray.points(P, valid=pv)), ctx.upload(GeoArrowArray.points(Q))
    d, valid = engine.haversine_distance(a, b)
    empty = (np.isnan(P).all(axis=1)) | (np.isnan(Q).all(axis=1))
    assert np.array_equal(valid.astype(bool), pv & ~empty) and np.all(np.isnan(d[~valid.astype(bool)]))
    assert valid[-2] and np.isnan(d[-2]) and valid[-1] and np.isnan(d[-1])  # a non-finite coordinate: what the expression gives
    # == geodesic_length("haversine") of the two-point linestring, bit for bit
    xy = np.empty((2 * len(P), 2))
    xy[0::2], xy[1::2] = P, Q
    ls = ctx.upload(GeoArrowArray.linestrings(xy, np.arange(0, 2 * len(P) + 1, 2, dtype=np.int64)))
    gl, _ = engine.geodesic_length(ls, "haversine")
    ok = valid.astype(bool)
    assert same_f64(d[ok], gl[ok])
    want = gref.haversine(P, Q)
    fin = ok & ~np.isnan(want) & ~np.isnan(d)
    assert fin.sum() >= 2800
    near_antipode = want > HALF * (1 - 1e-4)  # a > 1 - 1e-9 or so: asin is ill-conditioned, compare absolutely
    assert np.all(np.abs(d[fin & ~near_antipode] - want[fin & ~near_antipode]) <= 1e-9 * np.maximum(want[fin & ~near_antipode], 1e-3))
    assert np.all(np.abs(d[fin & near_antipode] - want[fin & near_antipode]) <= 1.0)
    assert abs(d[3000] - R * math.pi / 2) < 1e-6 and abs(d[3002] - 0.2 * math.pi / 180 * R) < 1e-6
    # the GeoSeries accessor gives the same values, nulls where a point is null or empty
    s = GeoSeries(_device=a).geo.haversine_distance(GeoSeries(_device=b))
    assert s.null_count == int((~ok).sum()) and same_f64(np.asarray(s.fill_null(0.0))[ok], d[ok])
    with pytest.raises(_lib.MismatchedGeometry):
        engine.haversine_distance(a, ls)
    with pytest.raises(_lib.ShapeError):
        engine.haversine_distance(a, ctx.upload(GeoArrowArray.points(Q[:5])))


@pytest.mark.parametrize("D", [0.0, 1.0, 3e4, 5e5, 1.0 * R * 0.99, 1.0 * R * 1.01, HALF])
def test_joins_vs_referee_with_planted_rows(ctx, D):
    L, lv, Rr, rv = fixture(np.random.default_rng(2), 80, 1500)
    idx = check(ctx, L, Rr, D, lvalid=lv, rvalid=rv)
    assert idx.stats()["ineligible"] >= 8
    check(ctx, L, Rr, None, maxd=D, lvalid=lv, rvalid=rv, cpu=False)


def test_antimeridian_in_both_conventions(ctx):
    rng = np.random.default_rng(3)
    east = np.column_stack([rng.uniform(179.5, 180.0, 200), rng.uniform(-1, 1, 200)])
    west = np.column_stack([rng.uniform(-180.0, -179.5, 200), rng.uniform(-1, 1, 200)])
    Rr = np.concatenate([east, west, [[179.9, 0.0], [-179.9, 0.0], [180.0, 0.0], [-180.0, 0.0]]])
    L = np.concatenate([Rr[::9], [[179.9, 0.0], [-179.9, 0.0], [math.nextafter(180.0, 0.0), 0.0], [-180.0, 0.5]]])
    out = []
    for conv in (lambda X: X, lambda X: np.column_stack([np.where(X[:, 0] < 0, X[:, 0] + 360.0, X[:, 0]), X[:, 1]])):
        idx = check(ctx, conv(L), conv(Rr), 3e4)
        ld = ctx.upload(GeoArrowArray.points(conv(L)))
        out.append(idx.count_within(ld, 3e4))
        d = engine.haversine_distance(ctx.upload(GeoArrowArray.points(conv(L[-4:-3]))), ctx.upload(GeoArrowArray.points(conv(Rr[401:402]))))[0][0]
        assert abs(d - 0.2 * math.pi / 180 * R) < 1e-6  # (179.9, 0) to (-179.9, 0): 22 km, not 359.8 degrees
    assert out[0][-4] > 20 and np.abs(out[0].astype(int) - out[1]).max() <= 1  # the same neighbours either way (up to an ulp at D)
    check(ctx, L, np.column_stack([np.where(Rr[:, 0] < 0, Rr[:, 0] + 360.0, Rr[:, 0]), Rr[:, 1]]), 3e4)  # conventions mixed


def test_poles(ctx):
    rng = np.random.default_rng(4)
    north = np.column_stack([rng.uniform(-180, 180, 300), 90.0 - np.abs(rng.normal(0, 0.05, 300))])
    south = np.column_stack([rng.uniform(0, 360, 300), -90.0 + np.abs(rng.normal(0, 0.05, 300))])
    Rr = np.concatenate([north, south, [[0.0, 90.0], [120.0, 90.0], [5.0, -90.0]]])
    L = np.array([[0.0, 90.0], [77.0, 90.0], [-140.0, 89.99], [10.0, -90.0], [200.0, -89.95], [0.0, 0.0], [33.0, math.nextafter(90.0, 0.0)]])
    for D in (0.0, 1e3, 8e3, 3e4):
        check(ctx, L, Rr, D)
    idx = engine.GeoIndex(ctx.upload(GeoArrowArray.points(Rr)))
    assert idx.count_within(ctx.upload(GeoArrowArray.points(L[:1])), 3e4)[0] > 250  # rows at every longitude around the pole


def test_D_zero_duplicates_boundary_and_invalid_arguments(ctx):
    Rr = np.array([[10.0, 20.0], [10.0, 20.0], [12.0, 20.0], [8.0, 20.0], [10.0, 21.0], [370.0 - 360.0, 20.0]])
    L = np.array([[10.0, 20.0], [10.0, 20.5], [11.0, 20.0]])
    idx = check(ctx, L, Rr, 0.0)
    ld = ctx.upload(GeoArrowArray.points(L))
    assert idx.count_within(ld, 0.0).tolist() == [3, 0, 0]
    nid, dist, tied = idx.query(ld)
    assert nid[0] == 0 and dist[0] == 0.0 and tied[0] == 3
    # lattice ties: mirrored longitudes at one latitude
    d_e = engine.haversine_distance(ctx.upload(GeoArrowArray.points(L[:1])), ctx.upload(GeoArrowArray.points(Rr[2:3])))[0][0]
    a, b, d = idx.pairs_within(ld, d_e, with_distance=True)
    row0 = b[a == 0].tolist()
    assert 2 in row0 and 3 in row0 and d[(a == 0) & (b == 2)][0] == d[(a == 0) & (b == 3)][0] == d_e  # D at a pair's distance: kept
    a, b = idx.pairs_within(ld, math.nextafter(d_e, 0.0))
    assert 2 not in b[a == 0].tolist() and 3 not in b[a == 0].tolist()  # one ulp below: dropped
    check(ctx, L, Rr, d_e)
    # max_distance at the nearest distance, one ulp below, 0 and inf
    d1 = idx.query(ld)[1][1]
    assert idx.query(ld, d1)[0][1] >= 0 and idx.query(ld, math.nextafter(d1, 0.0))[0][1] == -1
    assert idx.query(ld, 0.0)[0].tolist() == [0, -1, -1] and idx.query(ld, INF)[0][1] >= 0
    for bad in (math.nan, -1.0, INF, -INF):
        with pytest.raises(_lib.GeopolarsError) as e:
            idx.count_within(ld, bad)
        assert e.value.code == -7
        with pytest.raises(_lib.GeopolarsError):
            idx.pairs_within(ld, bad)
    for bad in (math.nan, -1.0, -INF):
        with pytest.raises(_lib.GeopolarsError) as e:
            idx.query(ld, bad)
        assert e.value.code == -7
        with pytest.raises(_lib.GeopolarsError):
            idx.pairs(ld, bad)
    ls = ctx.upload(GeoArrowArray.from_shapes(GeometryType.LINESTRING, [[(0, 0), (1, 1)]]))
    with pytest.raises(_lib.MismatchedGeometry):
        engine.GeoIndex(ls)
    for call in (lambda: idx.count_within(ls, 1.0), lambda: idx.pairs_within(ls, 1.0), lambda: idx.query(ls), lambda: idx.pairs(ls)):
        with pytest.raises(_lib.MismatchedGeometry):
            call()


def test_degenerate_right_sides(ctx):
    rng = np.random.default_rng(5)
    L = np.concatenate([sphere(rng, 40), [[179.9, 10.0], [-179.9, 10.0], [30.0, 0.0]]])
    one = np.array([[179.95, 10.0]])
    meridian = np.column_stack([np.full(50, 180.0), np.linspace(-80, 80, 50)])
    parallel = np.column_stack([np.linspace(-180, 179, 60), np.zeros(60)])
    for Rr, shape in ((one, (1, 1)), (meridian, (1, None)), (parallel, (None, 1))):
        for D in (0.0, 2e4, 2e6, HALF):
            idx = check(ctx, L, Rr, D)
        st = idx.stats()
        assert (shape[0] is None or st["grid_columns"] == shape[0]) and (shape[1] is None or st["grid_rows"] == shape[1])
    # a right column that is all null, one that is all out of range, and an empty one
    for Rr, rv in ((sphere(rng, 20), np.zeros(20, bool)), (np.column_stack([np.full(5, 400.0), np.zeros(5)]), None), (np.zeros((0, 2)), None)):
        idx = check(ctx, L, Rr, 1e6, rvalid=rv)
        assert idx.stats()["rows"] == 0
    check(ctx, np.zeros((0, 2)), sphere(rng, 20), 1e6)


def test_bundled_datasets(ctx):
    from geopolars_b200 import datasets

    cities = datasets.read_dataset("cities").geometry.device.to_host()
    ne = datasets.read_dataset("naturalearth_cities").geometry.device.to_host()
    assert cities.type == GeometryType.POINT and ne.type == GeometryType.POINT
    for D in (5e4, 5e5):
        check(ctx, cities.xy, ne.xy, D, lvalid=cities.valid, rvalid=ne.valid)
        check(ctx, ne.xy, ne.xy, D, lvalid=ne.valid, rvalid=ne.valid)
    nid, dist, _ = engine.GeoIndex(ctx.upload(ne)).query(ctx.upload(ne))
    assert np.array_equal(nid[dist == 0.0], np.arange(len(ne))[dist == 0.0]) or (dist == 0.0).all()
    # the Python joins: how = inner / left
    lhs, rhs = GeoSeries(_device=ctx.upload(cities)), GeoSeries(_device=ctx.upload(ne))
    a, b, d = geo_dwithin_join(lhs, rhs, 1e5)
    la, lb, ldist = geo_dwithin_join(lhs, rhs, 1e5, how="left")
    assert len(la) == len(a) + len(set(range(len(lhs))) - set(a.tolist())) and (lb == -1).sum() == len(la) - len(a)
    assert np.all(np.isnan(ldist[lb == -1])) and same_f64(ldist[lb >= 0], d) and np.all(d <= 1e5)
    a, b, d = geo_nearest_join(lhs, rhs, max_distance=2e5)
    la, lb, ldist = geo_nearest_join(lhs, rhs, how="left", max_distance=2e5)
    assert set(la.tolist()) == set(range(len(lhs))) and np.array_equal(la[lb >= 0], a) and np.all(d <= 2e5)
    assert len(geo_nearest_join(lhs, rhs)[0]) >= len(lhs)
    with pytest.raises(ValueError):
        geo_nearest_join(lhs, rhs, how="outer")


def test_grid_cap_and_a_point_with_a_million_matches(ctx):
    rng = np.random.default_rng(6)
    Rr = sphere(rng, 4_300_000)
    Rr[:1_000_000] = np.column_stack([20.0 + rng.uniform(-0.05, 0.05, 1_000_000), 40.0 + rng.uniform(-0.05, 0.05, 1_000_000)])
    L = np.concatenate([[[20.0, 40.0]], sphere(rng, 2000)])
    idx = check(ctx, L, Rr, 2e4, sample=[0, 1, 2, 3, 1000], cpu=False)
    st = idx.stats()
    assert st["grid_cells_per_axis"] == 2048 and st["rows"] == 4_300_000
    ld = ctx.upload(GeoArrowArray.points(L))
    cnt = idx.count_within(ld, 2e4)
    assert cnt[0] >= 1_000_000
    a, b, d = idx.pairs_within(ld, 2e4, with_distance=True)
    a2, b2, d2 = idx.pairs_within(ld, 2e4, with_distance=True)
    assert a.tobytes() == a2.tobytes() and b.tobytes() == b2.tobytes() and d.tobytes() == d2.tobytes()  # byte-identical reruns
    n1, d1, t1 = idx.query(ld)
    n2, d2, t2 = idx.query(ld)
    assert n1.tobytes() == n2.tobytes() and d1.tobytes() == d2.tobytes() and t1.tobytes() == t2.tobytes()


def test_ten_million_by_one_million_vs_tree_candidates(ctx):
    """10 M x 1 M points uniform on the sphere at D = 10 km; a 1 M left slice is checked bit for bit against cKDTree
    candidates evaluated through gpl_haversine_distance"""
    from scipy.spatial import cKDTree

    rng = np.random.default_rng(7)
    Rr, L = sphere(rng, 1_000_000), sphere(rng, 10_000_000, -180.0, 360.0)
    D = 1e4
    rhs_dev, ld = ctx.upload(GeoArrowArray.points(Rr)), ctx.upload(GeoArrowArray.points(L))
    idx = engine.GeoIndex(rhs_dev)
    cnt = idx.count_within(ld, D)
    a, b, d = idx.pairs_within(ld, D, with_distance=True)
    assert len(a) == int(cnt.sum()) and np.array_equal(np.bincount(a.astype(np.int64), minlength=len(L)), cnt)
    n = 1_000_000
    cand = cKDTree(gref.unit(Rr)).query_ball_point(gref.unit(L[:n]), gref.chord(D / R), workers=-1)
    li = np.repeat(np.arange(n), [len(c) for c in cand])
    rj = np.concatenate([np.asarray(c, np.int64) for c in cand if len(c)])
    dd, _ = engine.haversine_distance(ctx.upload(GeoArrowArray.points(L[li])), ctx.upload(GeoArrowArray.points(Rr[rj])))
    keep = dd <= D
    order = np.lexsort((rj[keep], li[keep]))
    m = int(cnt[:n].sum())
    assert m == int(keep.sum()) and np.array_equal(a[:m].astype(np.int64), li[keep][order]) and np.array_equal(b[:m].astype(np.int64), rj[keep][order])
    assert same_f64(d[:m], dd[keep][order])
    # nearest on the same data: the distance equals the minimum over the tree's candidates wherever a row lies within D
    nid, dist, _ = idx.query(ctx.upload(GeoArrowArray.points(L[:n])), D)
    assert np.array_equal(nid >= 0, cnt[:n] > 0)
    has = np.nonzero(cnt[:n] > 0)[0]
    starts = np.concatenate([[0], np.cumsum(cnt[:n].astype(np.int64))])
    assert same_f64(dist[has], np.minimum.reduceat(d[:m], starts[has]))


def test_left_row_guard(ctx):
    """2^31 left rows (and right rows) are refused before any access: a Point array wrapped around a small buffer"""
    import ctypes as C

    import torch

    small = torch.zeros(16, dtype=torch.float64, device="cuda")
    big = ctx.wrap_device(GeometryType.POINT, 1 << 31, 1 << 31, small.data_ptr(), keepalive=(small,))
    idx = engine.GeoIndex(ctx.upload(GeoArrowArray.points(np.array([[0.0, 0.0]]))))
    buf = np.zeros(8, np.int32)
    h = C.c_void_p()
    assert ctx.lib.gpl_geo_dwithin_count(ctx._h, idx._h, big._h, 1.0, C.c_void_p(buf.ctypes.data), engine.GPL_DEVICE) == -6
    assert ctx.lib.gpl_geo_dwithin_join_pairs(ctx._h, idx._h, big._h, 1.0, 1, C.byref(h)) == -6
    assert ctx.lib.gpl_geo_nearest_join(ctx._h, idx._h, big._h, 1.0, C.c_void_p(buf.ctypes.data), None, None, engine.GPL_DEVICE) == -6
    assert ctx.lib.gpl_geo_nearest_join_pairs(ctx._h, idx._h, big._h, 1.0, C.byref(h), None, engine.GPL_DEVICE) == -6
    assert ctx.lib.gpl_geo_index_build(ctx._h, big._h, C.byref(h)) == -6
