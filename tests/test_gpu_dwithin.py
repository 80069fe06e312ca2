"""Distance-within join (gpl_dwithin_*, DESIGN.md §4.14): every right row within D of each left row.  The pair list is
compared bit for bit with a referee built from the row-wise `distance` entry point: for a sampled left row the referee
evaluates `distance(lhs, rhs)` on a column of that row repeated once per right row (the left row first) and keeps the right
rows in R with a non-null distance <= D.  The list must hold exactly those rows, sorted, with their distances bit for bit, and
its per-row lengths must equal `count_within`."""
import math
import time

import numpy as np
import pytest

import nearest_geom_reference as ngr
import shapes
from geopolars_b200 import GeoArrowArray, GeometryType, _lib, engine
from geopolars_b200.geoseries import GeoSeries, dwithin_join
from test_gpu_nearest import T, r_mask, same_f64
from test_gpu_nearest_geom import repeat_row, rows_of, to_og

pytestmark = pytest.mark.gpu

KINDS = list(T)


def referee_rows(ctx, lhs, rhs, rhs_dev, i, D, L=None, R=None):
    """(rows, distances) of the right rows within D of left row i, by brute force through `distance`"""
    L = r_mask(lhs) if L is None else L
    R = r_mask(rhs) if R is None else R
    m = len(rhs)
    if not L[i] or m == 0:
        return np.zeros(0, np.int64), np.zeros(0)
    d, valid = engine.distance(ctx.upload(repeat_row(lhs, i, m)), rhs_dev)
    js = np.nonzero(R & valid.astype(bool) & (d <= D))[0]
    return js, d[js]


def check_dwithin(ctx, lhs, rhs, D, sample=None, idx=None, cpu=True):
    """pair list == referee on `sample`, sorted, lengths == count_within; returns (idx, a, b, d, cnt)"""
    rhs_dev = ctx.upload(rhs)
    idx = idx or engine.NearestIndex(rhs_dev)
    ld = ctx.upload(lhs)
    cnt = idx.count_within(ld, D)
    a, b, d = idx.pairs_within(ld, D, with_distance=True)
    key = a.astype(np.int64) * (1 << 32) + b.astype(np.int64)
    assert np.all(np.diff(key) > 0)
    assert len(a) == int(cnt.sum())
    assert np.array_equal(np.bincount(a.astype(np.int64), minlength=len(lhs)), cnt)
    starts = np.concatenate([[0], np.cumsum(cnt.astype(np.int64))])
    sample = np.arange(len(lhs)) if sample is None else np.asarray(sample)
    L, R = r_mask(lhs), r_mask(rhs)
    for i in sample:
        js, dj = referee_rows(ctx, lhs, rhs, rhs_dev, i, D, L, R)
        assert np.array_equal(b[starts[i]:starts[i + 1]].astype(np.int64), js), i
        assert same_f64(d[starts[i]:starts[i + 1]], dj), i
    if cpu and len(rhs) * len(sample) <= 100_000:  # the CPU oracle's distances, away from the D boundary
        ol, orr = to_og(lhs), to_og(rhs)
        for i in sample:
            if not L[i]:
                continue
            od = ngr._dist(ol, i, orr, np.arange(len(rhs)))
            near = np.abs(od - D) <= 1e-9 * max(D, 1.0)
            want = np.nonzero(R & ~np.isnan(od) & (od <= D) & ~near)[0]
            got = b[starts[i]:starts[i + 1]].astype(np.int64)
            got_d = d[starts[i]:starts[i + 1]]
            keep = ~near[got]
            assert np.array_equal(got[keep], want), i
            from conftest import rel_close

            assert rel_close(got_d, od[got])
    return idx, a, b, d, cnt


def left_rows(kind, rng, n):
    if kind == "point":
        P = np.concatenate([rng.uniform(-2, 12, (n, 2)), [[np.nan, 1.0], [1e6, 0.0]]])
        pv = np.ones(len(P), bool)
        pv[::7] = False
        return GeoArrowArray.points(P, valid=pv)
    rows = shapes.random_rows(rng, kind, n) + ngr.planted(kind)
    return GeoArrowArray.from_shapes(T[kind], [rows[i] for i in rng.permutation(len(rows))])


@pytest.mark.parametrize("lk", KINDS)
@pytest.mark.parametrize("rk", KINDS)
def test_every_type_pair_vs_referee(ctx, lk, rk):
    rng = np.random.default_rng(100 + KINDS.index(lk) * 6 + KINDS.index(rk))
    rhs = GeoArrowArray.from_shapes(T[rk], rows_of(rk, rng, 100))
    lhs = left_rows(lk, rng, 30)
    for D in (0.0, 0.7, 3.0):
        idx, a, _, _, cnt = check_dwithin(ctx, lhs, rhs, D)
    assert idx.stats()["evaluations"] > 0 and idx.stats()["overflow_points"] == 0
    assert (cnt[~r_mask(lhs)] == 0).all()


def test_distance_edges_and_invalid_distances(ctx):
    sq = lambda x, y, s: [[(x, y), (x + s, y), (x + s, y + s), (x, y + s), (x, y)]]
    rhs = GeoArrowArray.from_shapes(GeometryType.POLYGON, [sq(float(x), float(y), 1.0) for x in range(10) for y in range(10)])
    # touching (shared edge / corner) and overlapping rows: D = 0 keeps exactly the rows at distance 0
    lhs = GeoArrowArray.from_shapes(GeometryType.POLYGON, [sq(2.0, 2.0, 1.0), sq(4.5, 4.5, 0.25), sq(20.0, 20.0, 1.0)])
    _, a, b, d, cnt = check_dwithin(ctx, lhs, rhs, 0.0)
    assert cnt[0] == 9 and cnt[1] == 1 and cnt[2] == 0 and (d == 0.0).all()
    # D equal to a planted pair's distance includes it, one ulp below excludes it
    rng = np.random.default_rng(4)
    segs = GeoArrowArray.from_shapes(GeometryType.LINESTRING, shapes.random_rows(rng, "linestring", 40, span=30.0))
    rd = ctx.upload(rhs)
    dd, _ = engine.distance(ctx.upload(repeat_row(segs, 5, len(rhs))), rd)
    dk = float(np.sort(dd)[3])
    idx = engine.NearestIndex(rd)
    _, a1, b1, _, _ = check_dwithin(ctx, segs, rhs, dk, idx=idx, sample=np.r_[5, 0:8])
    _, a2, b2, _, _ = check_dwithin(ctx, segs, rhs, float(np.nextafter(dk, 0.0)), idx=idx, sample=np.r_[5, 0:8])
    j = int(np.nonzero(dd == dk)[0][0])
    assert ((a1 == 5) & (b1 == j)).any() and not ((a2 == 5) & (b2 == j)).any()
    ld = ctx.upload(segs)
    for bad in (math.nan, -1.0, math.inf, -math.inf):
        with pytest.raises(_lib.GeopolarsError) as e:
            idx.count_within(ld, bad)
        assert e.value.code == -7
        with pytest.raises(_lib.GeopolarsError) as e:
            idx.pairs_within(ld, bad)
        assert e.value.code == -7


def test_slack_keeps_pairs_computed_below_their_box_distance(ctx):
    """D between the computed distance of a left segment to a long segment and their box distance (the case
    test_nearest_geom_bound_model.py's tau = 0 control finds): only the slack keeps the pair"""
    from test_nearest_geom_bound_model import slack_cases

    for p, Lx, dB, fill in slack_cases(2):
        rows = [[(0.0, 0.0), (Lx, 0.0)], [(p[0] - dB, p[1]), (p[0] - dB, p[1] + 1.0)]] + fill
        rhs = GeoArrowArray.from_shapes(GeometryType.LINESTRING, rows)
        lhs = GeoArrowArray.from_shapes(GeometryType.LINESTRING, [[p, (p[0], p[1] + 1.0)]])
        dA, _ = engine.distance(ctx.upload(lhs), ctx.upload(GeoArrowArray.from_shapes(GeometryType.LINESTRING, [rows[0]])))
        assert dA[0] < p[1]  # computed below the box distance p.y
        _, a, b, d, cnt = check_dwithin(ctx, lhs, rhs, float(dA[0]), cpu=False)
        assert cnt[0] == 1 and b[0] == 0 and d[0] == dA[0]
    # the same with a Point left side: (0.5, 1) against (0, 0)-(49, 0) computes 1 ulp below its box distance 1
    rhs = GeoArrowArray.from_shapes(GeometryType.LINESTRING, [[(0.0, 0.0), (49.0, 0.0)]] + [[(x, 5.0), (x + 0.5, 5.0)] for x in range(0, 48, 2)])
    lhs = GeoArrowArray.points(np.array([[0.5, 1.0]]))
    _, a, b, d, cnt = check_dwithin(ctx, lhs, rhs, 0.9999999999999999, cpu=False)
    assert cnt[0] == 1 and b[0] == 0


def test_window_edge_row_is_evaluated(ctx):
    """a right point whose designated cell lies just past fl(p.x - (D + tau)) because the gap rounds down to D + tau
    (tests/test_dwithin_window_model.py::edge_case): with the margin it is a candidate and evaluated; without it, it is not"""
    from test_dwithin_window_model import edge_case

    p, q, D = edge_case()
    rhs = GeoArrowArray.points(np.array([[-500.0, -500.0], [500.0, 500.0], list(q)]))
    idx = engine.NearestIndex(ctx.upload(rhs))
    assert idx.stats()["grid_cells_per_axis"] == 2
    cnt = idx.count_within(ctx.upload(GeoArrowArray.points(np.array([list(p)]))), D)
    assert cnt[0] == 0 and idx.stats()["evaluations"] == 1


def test_regimes(ctx):
    """zero-width / zero-height right boxes, left rows 1e6 outside the grid, a right row spanning the whole grid"""
    rng = np.random.default_rng(5)
    flat = [[(x, 0.0), (x + 0.5, 0.0)] for x in np.sort(rng.uniform(0, 100, 300))]
    tall = GeoArrowArray.points(np.stack([np.full(300, 2.5), rng.uniform(0, 10, 300)], 1))
    span = flat + [[(-10.0, -10.0), (110.0, 50.0)]]
    left = GeoArrowArray.from_shapes(GeometryType.POLYGON, shapes.random_rows(rng, "polygon", 30, span=100.0) +
                                     [[[(1e6, 5.0), (1e6 + 1.0, 5.0), (1e6, 6.0), (1e6, 5.0)]]])
    check_dwithin(ctx, left, GeoArrowArray.from_shapes(GeometryType.LINESTRING, span), 2.0)
    check_dwithin(ctx, left, tall, 2.0)
    P = np.concatenate([rng.uniform(-5, 105, (60, 2)), [[1e6, 0.0], [-1e6, 1e6], [2.5, 5.0]]])
    check_dwithin(ctx, GeoArrowArray.points(P), GeoArrowArray.from_shapes(GeometryType.LINESTRING, span), 1.5)
    check_dwithin(ctx, GeoArrowArray.points(P), tall, 1e6 + 10.0, sample=np.r_[0:5, 60:63], cpu=False)


def test_grid_cap(ctx):
    """4.3 M right points: the index reaches the 2048-cell cap"""
    import torch

    n = 4_300_000
    xy = torch.empty((n, 2), dtype=torch.float64, device="cuda")
    engine.check(ctx.lib.gpl_gen_uniform_points(ctx._h, 9, 0, n, 1000.0, xy.data_ptr()))
    ctx.synchronize()
    rhs = GeoArrowArray.points(xy.cpu().numpy())
    rd = ctx.upload(rhs)
    idx = engine.NearestIndex(rd)
    assert idx.stats()["grid_cells_per_axis"] == 2048
    rng = np.random.default_rng(2)
    lines = GeoArrowArray.from_shapes(GeometryType.LINESTRING, [[tuple(p), tuple(p + rng.uniform(-0.5, 0.5, 2))] for p in rng.uniform(-1, 1001, (6, 2))])
    check_dwithin(ctx, lines, rhs, 0.3, idx=idx, cpu=False)
    pts = GeoArrowArray.points(np.concatenate([rng.uniform(-1, 1001, (6, 2)), [[5e5, 5e5]]]))
    check_dwithin(ctx, pts, rhs, 0.5, idx=idx, cpu=False)


def test_queue_drains_and_resumes(ctx):
    """one left polygon with 3 000+ matching right polygons (the warp queue drained many times), and a point tile where every
    lane has hundreds of candidates (the shared 256-pair queue drained many times in one tile)"""
    rng = np.random.default_rng(11)
    rows = [[shapes.star_ring(rng, *rng.uniform(40, 60, 2), 5.0, 6, q=3)] for _ in range(3000)]
    rows += [[shapes.star_ring(rng, *rng.uniform(-100, 200, 2), 2.0, 6, q=3)] for _ in range(300)]
    rhs = GeoArrowArray.from_shapes(GeometryType.POLYGON, rows)
    lhs = GeoArrowArray.from_shapes(GeometryType.POLYGON, [[[(30.0, 30.0), (70.0, 30.0), (70.0, 70.0), (30.0, 70.0), (30.0, 30.0)]]])
    _, _, _, _, cnt = check_dwithin(ctx, lhs, rhs, 0.5, cpu=False)
    assert cnt[0] >= 3000
    pts = GeoArrowArray.points(rng.uniform(0, 10, (20_000, 2)))
    left = GeoArrowArray.points(rng.uniform(4, 6, (64, 2)))
    idx, _, _, _, cnt = check_dwithin(ctx, left, pts, 1.0, cpu=False)
    assert (cnt >= 400).all()
    polys = GeoArrowArray.from_shapes(GeometryType.POLYGON, [[shapes.star_ring(rng, *rng.uniform(0, 10, 2), 0.2, 6, q=3)] for _ in range(3000)])
    _, _, _, _, cnt = check_dwithin(ctx, left, polys, 1.0, sample=np.arange(0, 64, 4), cpu=False)
    assert (cnt >= 50).all()


def test_everywhere_rows_on_both_sides(ctx):
    sq = lambda x, y: [(x, y), (x + 1, y), (x + 1, y + 1), (x, y + 1), (x, y)]
    rng = np.random.default_rng(3)
    rrows = [[[sq(x, y)]] for x, y in rng.uniform(0, 50, (300, 2))] + [[[sq(80.0, 80.0)], []]]
    rhs = GeoArrowArray.from_shapes(GeometryType.MULTIPOLYGON, rrows)
    lrows = [[[(x, y), (x + 0.2, y + 0.1)]] for x, y in rng.uniform(0, 50, (40, 2))] + [[[(3.0, 3.0)], [(9.0, 9.0), (9.5, 9.0)]], [[], [(1.0, 1.0), (2.0, 2.0)]]]
    lhs = GeoArrowArray.from_shapes(GeometryType.MULTILINESTRING, lrows)
    check_dwithin(ctx, lhs, rhs, 2.0)
    rl = GeoArrowArray.from_shapes(GeometryType.LINESTRING, [[(float(x), float(y)), (x + 0.5, y + 0.5)] for x, y in rng.uniform(0, 50, (200, 2))] +
                                   [[(20.0, 20.0)], [(70.0, 70.0)]])
    lm = GeoArrowArray.from_shapes(GeometryType.MULTIPOINT, [[(20.0 + 1e-7, 20.0)], [(70.0, 70.0 - 5e-8), (60.0, 60.0)], [(100.0, 100.0)],
                                                              [(25.0, 25.0), (20.0, 20.0)]])
    idx, a, b, _, _ = check_dwithin(ctx, lm, rl, 0.0)
    assert idx.stats()["everywhere"] == 2 and ((a == 0) & (b == 200)).any() and ((a == 1) & (b == 201)).any()


def test_segment_sizes_and_a_million_matches(ctx, capsys):
    """per-row segments of 0, 1, 31-33, around the on-chip sort limit (256) and beyond, and one point matching 10^6 points"""
    xs = np.arange(3000, dtype=np.float64)
    rhs = GeoArrowArray.points(np.stack([xs[np.random.default_rng(0).permutation(3000)], np.zeros(3000)], 1))
    idx = engine.NearestIndex(ctx.upload(rhs))
    for s in (0, 1, 31, 32, 33, 255, 256, 257, 1000, 2999):
        # at (1500, 0) radius r keeps 2r + 1 lattice points; at (1500.5, 0) radius r - 0.5 keeps 2r
        r = s // 2
        x, D = (1500.0, float(r)) if s % 2 else (1500.5, r - 0.5 if r else 0.25)
        _, a, b, d, cnt = check_dwithin(ctx, GeoArrowArray.points(np.array([[x, 0.0], [1e5, 0.0]])), rhs, D, idx=idx, sample=[0], cpu=False)
        assert cnt[0] == s and cnt[1] == 0
    import torch

    n = 1_000_000
    xy = torch.empty((n, 2), dtype=torch.float64, device="cuda")
    engine.check(ctx.lib.gpl_gen_uniform_points(ctx._h, 21, 0, n, 1.0, xy.data_ptr()))
    ctx.synchronize()
    big = GeoArrowArray.points(xy.cpu().numpy())
    bd = ctx.upload(big)
    idx = engine.NearestIndex(bd)
    left = ctx.upload(GeoArrowArray.points(np.array([[0.5, 0.5], [0.25, 0.75]])))
    idx.pairs_within(left, 1.0)  # warm
    t = time.perf_counter()
    a, b, d = idx.pairs_within(left, 1.0, with_distance=True)
    dt = time.perf_counter() - t
    assert int((a == 0).sum()) == n
    js, dj = referee_rows(ctx, GeoArrowArray.points(np.array([[0.5, 0.5]])), big, bd, 0, 1.0)
    assert np.array_equal(b[a == 0].astype(np.int64), js) and same_f64(d[a == 0], dj)
    with capsys.disabled():
        print(f"\n[dwithin] one point x 10^6 matching points (+ a second point): pairs_within {dt * 1e3:.1f} ms for {len(a)} pairs")


def test_bundled_datasets(ctx):
    from geopolars_b200 import datasets

    cities = datasets.read_dataset("naturalearth_cities").geometry.device.to_host()
    countries = datasets.read_dataset("naturalearth_lowres").geometry.device.to_host()
    nybb = datasets.read_dataset("nybb").geometry.device.to_host()
    rng = np.random.default_rng(4)
    check_dwithin(ctx, countries, cities, 2.0, sample=rng.choice(len(countries), 30, replace=False), cpu=False)
    check_dwithin(ctx, nybb, nybb, 5000.0, cpu=False)


def test_ten_million_by_one_million_points(ctx):
    """10 M x 1 M uniform points in [0, 1000)^2, D = 1: the total of count_within is the pair count, and a 1 M left slice equals
    an independent CPU construction (cKDTree candidates at a larger radius, np.hypot distances, <= D) bit for bit"""
    import torch
    from scipy.spatial import cKDTree

    nl, nr_, D = 10_000_000, 1_000_000, 1.0
    lxy = torch.empty((nl, 2), dtype=torch.float64, device="cuda")
    rxy = torch.empty((nr_, 2), dtype=torch.float64, device="cuda")
    engine.check(ctx.lib.gpl_gen_uniform_points(ctx._h, 1, 0, nl, 1000.0, lxy.data_ptr()))
    engine.check(ctx.lib.gpl_gen_uniform_points(ctx._h, 2, 0, nr_, 1000.0, rxy.data_ptr()))
    ctx.synchronize()
    L, R = lxy.cpu().numpy(), rxy.cpu().numpy()
    idx = engine.NearestIndex(ctx.upload(GeoArrowArray.points(R)))
    ld = ctx.upload(GeoArrowArray.points(L))
    cnt = idx.count_within(ld, D)
    a, b, d = idx.pairs_within(ld, D, with_distance=True)
    assert len(a) == int(cnt.sum()) and 2.5e7 < len(a) < 3.8e7
    lo, hi = 3_000_000, 4_000_000
    s0, s1 = int(cnt[:lo].sum()), int(cnt[:hi].sum())
    ga, gb, gd = a[s0:s1].astype(np.int64), b[s0:s1].astype(np.int64), d[s0:s1]
    nb = cKDTree(R).query_ball_point(L[lo:hi], D * (1 + 1e-9) + 1e-12, workers=-1, return_sorted=True)
    ln = np.fromiter((len(x) for x in nb), np.int64, count=hi - lo)
    ca = np.repeat(np.arange(lo, hi), ln)
    cb = np.concatenate([np.asarray(x, np.int64) for x in nb])
    cd = np.hypot(R[cb, 0] - L[ca, 0], R[cb, 1] - L[ca, 1])
    k = cd <= D
    assert np.array_equal(ga, ca[k]) and np.array_equal(gb, cb[k]) and same_f64(gd, cd[k])


def test_nearest_join_cross_check(ctx):
    """1 M points x config 2's polygons: where nearest_join finds a row within D its distance is the minimum of the point's
    dwithin distances and its tied rows are among the point's dwithin rows; where it finds none, count_within is 0"""
    import torch

    from geopolars_b200 import synth

    pxy, ro, go = synth.star_polygons(10_000, 100, 10.0, 64)
    rd = ctx.upload(GeoArrowArray.polygons(pxy, ro, go))
    n, D = 1_000_000, 0.5
    xy = torch.empty((n, 2), dtype=torch.float64, device="cuda")
    engine.check(ctx.lib.gpl_gen_uniform_points(ctx._h, 5, 0, n, 1000.0, xy.data_ptr()))
    ctx.synchronize()
    ld = ctx.upload(GeoArrowArray.points(xy.cpu().numpy()))
    idx = engine.NearestIndex(rd)
    na, nb_, ndist = idx.pairs_array(ld, D, with_distance=True)
    cnt = idx.count_within(ld, D)
    a, b, d = idx.pairs_within(ld, D, with_distance=True)
    has = ~np.isnan(ndist)
    assert (cnt[~has] == 0).all() and (cnt[has] > 0).all()
    starts = np.concatenate([[0], np.cumsum(cnt.astype(np.int64))])
    rows = np.nonzero(has)[0]
    mins = np.minimum.reduceat(d, starts[rows])
    assert same_f64(mins, ndist[rows])
    dw = set(zip(a.tolist(), b.tolist()))
    assert all((int(i), int(j)) in dw for i, j in zip(na, nb_))


def test_accessor_guards_and_determinism(ctx):
    import ctypes as C

    import torch

    rng = np.random.default_rng(9)
    rhs = GeoArrowArray.from_shapes(GeometryType.POLYGON, shapes.random_rows(rng, "polygon", 100))
    lrows = shapes.random_rows(rng, "linestring", 60, span=14.0) + [None, [], [(np.nan, 1.0), (2.0, 2.0)]]
    lhs = GeoSeries(_device=ctx.upload(GeoArrowArray.from_shapes(GeometryType.LINESTRING, lrows)))
    rs = GeoSeries(_device=ctx.upload(rhs))
    idx = engine.NearestIndex(rs.device)
    a, b, d = dwithin_join(lhs, rs, 0.5)
    la, lb, ld_ = idx.pairs_within(lhs.device, 0.5, with_distance=True)
    assert np.array_equal(a, la) and np.array_equal(b, lb) and same_f64(d, ld_)
    assert not np.isin([60, 61, 62], a).any()
    a2, b2, d2 = dwithin_join(lhs, rs, 0.5, how="left")
    cnt = idx.count_within(lhs.device, 0.5)
    miss = np.nonzero(cnt == 0)[0]
    assert {60, 61, 62} <= set(miss.tolist())
    assert len(a2) == int(cnt.sum()) + len(miss) and sorted(set(a2.tolist())) == list(range(len(lrows)))
    assert (b2[np.isin(a2, miss)] == -1).all() and np.isnan(d2[np.isin(a2, miss)]).all()
    with pytest.raises(ValueError):
        dwithin_join(lhs, rs, 0.5, how="right")
    # row-wise dwithin == distance <= D, null distances False
    other = GeoSeries(_device=ctx.upload(GeoArrowArray.from_shapes(GeometryType.POLYGON, shapes.random_rows(rng, "polygon", len(lrows)))))
    dist, valid = engine.distance(lhs.device, other.device)
    got = np.asarray(lhs.geo.dwithin(other, 3.0).to_pylist())
    assert np.array_equal(got, valid.astype(bool) & (dist <= 3.0)) and not got[60]
    # two runs give byte-identical outputs
    x1 = idx.pairs_within(lhs.device, 2.0, with_distance=True)
    x2 = idx.pairs_within(lhs.device, 2.0, with_distance=True)
    assert all(u.tobytes() == v.tobytes() for u, v in zip(x1, x2))
    P = ctx.upload(GeoArrowArray.points(rng.uniform(0, 10, (5000, 2))))
    y1, y2 = idx.pairs_within(P, 1.0, with_distance=True), idx.pairs_within(P, 1.0, with_distance=True)
    assert all(u.tobytes() == v.tobytes() for u, v in zip(y1, y2))
    # 2^31 left rows: GPL_ERR_UNSUPPORTED before any access
    small = torch.zeros(16, dtype=torch.int64, device="cuda")
    big = ctx.wrap_device(GeometryType.LINESTRING, 1 << 31, 1 << 32, small.data_ptr(), geom_off_ptr=small.data_ptr(), keepalive=(small,))
    buf = np.zeros(8, np.int32)
    assert ctx.lib.gpl_dwithin_count(ctx._h, idx._h, big._h, 1.0, C.c_void_p(buf.ctypes.data), engine.GPL_DEVICE) == -6
    h = C.c_void_p()
    assert ctx.lib.gpl_dwithin_join_pairs(ctx._h, idx._h, big._h, 1.0, 1, C.byref(h)) == -6
    # a spatial_join result carries no distances
    h = C.c_void_p()
    engine.check(ctx.lib.gpl_spatial_join(ctx._h, rs.device._h, rs.device._h, 0, C.byref(h)))
    try:
        assert ctx.lib.gpl_pairs_count(h) > 0
        out = np.zeros(ctx.lib.gpl_pairs_count(h))
        assert ctx.lib.gpl_pairs_copy_distance(ctx._h, h, out.ctypes.data, engine.GPL_HOST) == -7
    finally:
        ctx.lib.gpl_pairs_free(h)
