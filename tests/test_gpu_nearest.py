"""Nearest-geometry join (gpl_nearest_*): every output is compared bit for bit with a referee built from the row-wise
`distance` entry point.  For a sampled point the referee evaluates `distance` on a column of that point repeated once
per right row, drops the rows outside the candidate set R (null, no envelope, a non-finite coordinate) and the rows
beyond max_distance, and takes the minimum, the lowest row at it and the number of rows at it."""
import math

import numpy as np
import pytest

import shapes
from geopolars_b200 import GeoArrowArray, GeometryType, _lib, engine
from geopolars_b200.geoseries import GeoSeries, nearest_join

pytestmark = pytest.mark.gpu

T = {
    "point": GeometryType.POINT,
    "multipoint": GeometryType.MULTIPOINT,
    "linestring": GeometryType.LINESTRING,
    "multilinestring": GeometryType.MULTILINESTRING,
    "polygon": GeometryType.POLYGON,
    "multipolygon": GeometryType.MULTIPOLYGON,
}
INF = float("inf")


# ---- the referee ------------------------------------------------------------------------------------------------------------
def _coord_ranges(a: GeoArrowArray):
    """per row: [c0, c1) over all its coordinates, and the number of coordinates envelope_raw counts (exterior rings)"""
    n, t = len(a), a.type
    r = np.arange(n)
    if t == GeometryType.POINT:
        c0, c1 = r, r + 1
        env = ~(np.isnan(a.xy[:, 0]) & np.isnan(a.xy[:, 1]))
        return c0, c1, env
    go = a.geom_off
    if t in (GeometryType.LINESTRING, GeometryType.MULTIPOINT):
        c0, c1 = go[:-1], go[1:]
        return c0, c1, c1 > c0
    ro = a.ring_off
    if t == GeometryType.MULTILINESTRING:
        c0, c1 = ro[go[:-1]], ro[go[1:]]
        return c0, c1, c1 > c0
    if t == GeometryType.POLYGON:
        c0, c1 = ro[go[:-1]], ro[go[1:]]
        ext = np.array([ro[go[i] + 1] - ro[go[i]] if go[i + 1] > go[i] else 0 for i in range(n)])
        return c0, c1, ext > 0
    po = a.part_off
    c0, c1 = ro[po[go[:-1]]], ro[po[go[1:]]]
    ext = np.array([sum(ro[po[q] + 1] - ro[po[q]] for q in range(go[i], go[i + 1]) if po[q + 1] > po[q]) for i in range(n)])
    return c0, c1, ext > 0


def r_mask(a: GeoArrowArray) -> np.ndarray:
    c0, c1, env = _coord_ranges(a)
    fin = np.isfinite(a.xy).all(axis=1)
    cf = np.concatenate([[0], np.cumsum(~fin)])
    ok = env & (cf[c1] - cf[c0] == 0)
    if a.valid is not None:
        ok &= a.valid
    return ok


def referee_distances(ctx, rhs_dev, m, p):
    col = ctx.upload(GeoArrowArray.points(np.tile(np.asarray(p, dtype=np.float64), (m, 1))))
    d, _ = engine.distance(col, rhs_dev)
    return d


def referee(ctx, rhs_host, rhs_dev, P, maxd=INF, R=None):
    """(nearest_id, distance, n_tied, {i: tied rows}) for the points P, by brute force through `distance`"""
    R = r_mask(rhs_host) if R is None else R
    m = len(rhs_host)
    nid, dist, tied, rows = [], [], [], {}
    for i, p in enumerate(P):
        if not (np.isfinite(p[0]) and np.isfinite(p[1])):
            nid.append(-1), dist.append(np.nan), tied.append(0)
            continue
        d = referee_distances(ctx, rhs_dev, m, p)
        ok = R & (d <= maxd)
        if not ok.any():
            nid.append(-1), dist.append(np.nan), tied.append(0)
            continue
        best = d[ok].min()
        js = np.nonzero(ok & (d == best))[0]
        nid.append(int(js[0])), dist.append(best), tied.append(len(js))
        rows[i] = js
    return np.array(nid, np.int32), np.array(dist), np.array(tied, np.int32), rows


def same_f64(a, b):
    return np.array_equal(np.asarray(a, np.float64).view(np.int64), np.asarray(b, np.float64).view(np.int64))


def check_join(ctx, rhs_host, P, maxd=INF, sample=None, pvalid=None, idx=None):
    """join outputs for all of P (+ pair list) == referee on `sample` rows; returns the index (for stats)"""
    rhs_dev = ctx.upload(rhs_host)
    idx = idx or engine.NearestIndex(rhs_dev)
    pts = GeoArrowArray.points(P, valid=pvalid)
    pd = ctx.upload(pts)
    nid, dist, tied = idx.query_array(pd, maxd)
    lhs, rhs = idx.pairs_array(pd, maxd)
    sample = np.arange(len(P)) if sample is None else sample
    Ps = P[sample].copy()
    if pvalid is not None:
        Ps[~pvalid[sample]] = np.nan  # null points match nothing, like non-finite ones
    rn, rd, rt, rows = referee(ctx, rhs_host, rhs_dev, Ps, maxd)
    assert np.array_equal(nid[sample], rn)
    assert same_f64(dist[sample], rd)
    assert np.array_equal(tied[sample], rt)
    # pair list: sorted, each tied row once, consistent with the dense form
    assert np.all(np.diff(lhs.astype(np.int64) * (1 << 32) + rhs.astype(np.int64)) > 0)
    assert len(lhs) == int(tied.sum())
    starts = np.searchsorted(lhs, np.arange(len(P)))
    for k, i in enumerate(sample):
        got = rhs[starts[i]:starts[i] + tied[i]].astype(np.int64)
        assert np.array_equal(got, rows.get(k, np.zeros(0, np.int64))), i
    if len(rhs_host) <= 20_000:
        oracle_agrees(rhs_host, P[sample], None if pvalid is None else pvalid[sample], maxd, nid[sample], dist[sample])
    # the pairs call hands back the same dense distances
    _, _, d3 = idx.pairs_array(pd, maxd, with_distance=True)
    assert same_f64(d3, dist)
    # the raw-coordinate entry point agrees where the points are valid
    if pvalid is None:
        n2, d2, t2 = idx.query(P, maxd)
        assert np.array_equal(n2, nid) and same_f64(d2, dist) and np.array_equal(t2, tied)
    return idx, nid, dist, tied


def oracle_agrees(rhs_host, P, pvalid, maxd, nid, dist):
    """the independent CPU reference (tests/nearest_reference.py, the oracle's distances, its own ring search): the
    distance within 1e-9, and the row wherever the best and second-best distances are more than 1e-9 apart"""
    import nearest_reference as nr
    from conftest import rel_close
    from oracle import oracle as og

    a = og.OGArray(int(rhs_host.type), rhs_host.xy, geom_off=rhs_host.geom_off, part_off=rhs_host.part_off, ring_off=rhs_host.ring_off,
                   valid=rhs_host.valid)
    rn, rd, _ = nr.nearest_join(a, P, pvalid, maxd, use_grid=True)
    R = nr.candidate_rows(a)[0]
    checked = 0
    for i in range(len(P)):
        if rn[i] < 0 and nid[i] < 0:
            continue
        b = rd[i] if rn[i] >= 0 else dist[i]
        if math.isfinite(maxd) and abs(b - maxd) <= 1e-9 * max(maxd, 1e-300):
            continue  # at the max_distance limit the two implementations may round to either side
        assert rn[i] >= 0 and nid[i] >= 0, i
        assert rel_close([dist[i]], [rd[i]]), (i, dist[i], rd[i])
        if nr.second_gap_ok(a, P[i], rd[i], R=R):
            assert nid[i] == rn[i], (i, nid[i], rn[i])
            checked += 1
    return checked


# ---- planted rows per type ----------------------------------------------------------------------------------------------------
def planted(kind, rng):
    """null, empty, NaN and 'everywhere' rows of one type that do not dominate the answer"""
    nan_pt = (math.nan, 3.0)
    if kind == "point":
        return [None, nan_pt, (math.nan, math.nan), (math.inf, 1.0)]
    if kind == "multipoint":
        return [None, [], [(1.0, 1.0), nan_pt]]
    if kind == "linestring":
        return [None, [], [(0.0, 0.0), nan_pt], [(4.05, 4.05)], [(7.3, 2.1)]]  # 1-coordinate rows: geo's point rule
    if kind == "multilinestring":
        return [None, [], [[(0.0, 0.0), (1.0, 1.0)], [(2.0, 2.0), nan_pt]], [[(3.3, 3.3)], [(8.0, 8.0), (9.0, 8.5)]]]
    if kind == "polygon":
        sq = [(2.0, 2.0), (3.0, 2.0), (3.0, 3.0), (2.0, 2.0)]
        return [None, [], [[(0.0, 0.0), (1.0, 0.0), nan_pt, (0.0, 0.0)]], [[(6.2, 6.2)]], [sq, [(20.0, 20.0)]]]
    sq = [(2.0, 2.0), (3.0, 2.0), (3.0, 3.0), (2.0, 2.0)]
    return [None, [], [[sq], [[(0.0, 0.0), nan_pt, (1.0, 1.0), (0.0, 0.0)]]], [[[(5.5, 5.5)]], [sq]], [[sq, [(30.0, -5.0), (31.0, -5.0)]]]]


def query_points(rng, n, span=10.0):
    P = np.concatenate([
        rng.uniform(-2, span + 2, (n, 2)),
        np.round(rng.uniform(0, span, (n // 4, 2)), 1),  # on the lattice of the shapes: vertices, edges, ties
        np.array([[1e6, 5.0], [-1e6, -1e6], [5.0, 2e6], [4.05, 4.05], [5.5, 5.5], [6.2, 6.2], [3.3, 3.3]]),
        np.array([[np.nan, 1.0], [np.inf, 0.0], [0.0, -np.inf]]),
    ])
    return P


@pytest.mark.parametrize("kind", list(T))
def test_every_type_vs_referee(ctx, kind):
    rng = np.random.default_rng(list(T).index(kind))
    rows = shapes.random_rows(rng, kind, 300) + planted(kind, rng)
    rows = [rows[i] for i in rng.permutation(len(rows))]
    rhs = GeoArrowArray.from_shapes(T[kind], rows)
    P = query_points(rng, 160)
    pvalid = np.ones(len(P), bool)
    pvalid[::17] = False
    idx, nid, dist, tied = check_join(ctx, rhs, P, pvalid=pvalid)
    st = idx.stats()
    R = r_mask(rhs)
    assert st["rows"] == int(R.sum()) and st["excluded"] == len(rhs) - int(R.sum())
    if kind not in ("point", "multipoint"):
        assert st["everywhere"] >= 1
    assert st["evaluations"] > 0
    # the far points still find their nearest row
    assert (nid[len(P) - 10:len(P) - 7] >= 0).all()


def test_everywhere_rows_tie_at_zero(ctx):
    """a row with an empty member has distance 0 from every point: it ties with every containing polygon"""
    rng = np.random.default_rng(3)
    sq = lambda x, y, s: [(x, y), (x + s, y), (x + s, y + s), (x, y + s), (x, y)]
    rows = [[[sq(x, y, 1.0)]] for x, y in rng.uniform(0, 50, (200, 2))] + [[[sq(0, 0, 1.0)], []], [[sq(0, 0, 1.0), []]]]
    rhs = GeoArrowArray.from_shapes(GeometryType.MULTIPOLYGON, rows)
    P = rng.uniform(-5, 55, (60, 2))
    idx, nid, dist, tied = check_join(ctx, rhs, P)
    assert idx.stats()["everywhere"] == 2
    assert (dist == 0.0).all() and (tied >= 2).all()


def test_lattice_ties(ctx):
    """points at the cell centres of a lattice of Point rows tie with the 4 corners; the pair list has each once"""
    g = np.arange(30, dtype=np.float64)
    X, Y = np.meshgrid(g, g)
    rhs = GeoArrowArray.points(np.stack([X.ravel(), Y.ravel()], 1))
    P = np.stack(np.meshgrid(np.arange(29) + 0.5, np.arange(29) + 0.5), -1).reshape(-1, 2)
    rng = np.random.default_rng(0)
    _, nid, dist, tied = check_join(ctx, rhs, P, sample=rng.choice(len(P), 120, replace=False))
    assert (tied == 4).all() and (dist == math.hypot(0.5, 0.5)).all()


def test_overlapping_polygons_and_overflow(ctx):
    """2 400 polygons around the same spot: points there tie at 0 with all of them (overflow path); a polygon that spans
    the whole grid ties with them"""
    rng = np.random.default_rng(11)
    rows = []
    for _ in range(2400):
        c = rng.uniform(45, 55, 2)
        rows.append(shapes.star_ring(rng, c[0], c[1], 30.0, 7, q=3))
    rows = [[r] for r in rows]
    rows.append([[(-100.0, -100.0), (200.0, -100.0), (200.0, 200.0), (-100.0, 200.0), (-100.0, -100.0)]])  # spans the grid
    rows += [[shapes.star_ring(rng, x, y, 2.0, 6, q=3)] for x, y in rng.uniform(-100, 200, (500, 2))]
    rhs = GeoArrowArray.from_shapes(GeometryType.POLYGON, rows)
    P = np.concatenate([rng.uniform(49, 51, (40, 2)), rng.uniform(-150, 250, (40, 2))])
    idx, nid, dist, tied = check_join(ctx, rhs, P, sample=np.r_[0:10, 40:60])
    assert idx.stats()["overflow_points"] >= 40
    assert tied[:40].min() > 1000 and (dist[:40] == 0).all()


def test_slack_keeps_rows_computed_below_their_box_distance(ctx):
    """a segment whose computed distance is below the distance to its box, and a point row just beyond it: the segment is
    the true nearest row, and only the slack tau keeps it from being pruned (DESIGN.md §4.12)"""
    from test_nearest_bound_model import line_segment_distance, pt_dist

    rng = np.random.default_rng(3)
    cases = []
    for _ in range(200_000):
        L = 10.0 ** rng.uniform(0, 3)
        p = (rng.uniform(0.1, L - 0.1), 10.0 ** rng.uniform(-1, 1))
        dA = line_segment_distance(p, (0.0, 0.0), (L, 0.0))
        dB = float(np.nextafter(dA, np.inf))
        q = (p[0] - dB, p[1])  # same y: its distance is the exact |dx| in every hypot
        if pt_dist(p, q) == dB and dB < p[1]:
            cases.append((p, L, q))
            if len(cases) == 8:
                break
    assert len(cases) == 8
    for p, L, q in cases:
        rhs = GeoArrowArray.from_shapes(GeometryType.LINESTRING, [[(0.0, 0.0), (L, 0.0)], [q, q]])
        _, nid, dist, tied = check_join(ctx, rhs, np.array([p]))
        assert nid[0] == 0 and tied[0] == 1 and dist[0] < p[1]


def test_max_distance(ctx):
    rng = np.random.default_rng(7)
    rows = shapes.random_rows(rng, "linestring", 200, span=100.0)
    rhs = GeoArrowArray.from_shapes(GeometryType.LINESTRING, rows)
    P = rng.uniform(-10, 110, (80, 2))
    rhs_dev = ctx.upload(rhs)
    idx = engine.NearestIndex(rhs_dev)
    _, d_all, _ = idx.query(P)
    k = int(np.argmax(d_all))
    dk = d_all[k]
    for maxd in (dk, np.nextafter(dk, 0.0), 0.0, INF, float(np.median(d_all))):
        check_join(ctx, rhs, P, maxd=maxd, sample=np.r_[k, 0:20], idx=idx)
    n1, d1, _ = idx.query(P, dk)
    n2, d2, _ = idx.query(P, np.nextafter(dk, 0.0))
    assert n1[k] >= 0 and n2[k] == -1 and np.isnan(d2[k])
    for bad in (math.nan, -1.0, -0.5e-300):
        with pytest.raises(_lib.GeopolarsError) as e:
            idx.query(P, bad)
        assert e.value.code == -7


def test_regimes(ctx):
    rng = np.random.default_rng(5)
    # one row
    one = GeoArrowArray.from_shapes(GeometryType.POLYGON, [shapes.random_polygon(rng)])
    idx, *_ = check_join(ctx, one, rng.uniform(-20, 30, (30, 2)))
    assert idx.stats()["grid_cells_per_axis"] == 1
    # zero-height union box: every row on y = 0
    xs = np.sort(rng.uniform(0, 100, 500))
    flat = GeoArrowArray.from_shapes(GeometryType.LINESTRING, [[(x, 0.0), (x + 0.5, 0.0)] for x in xs])
    check_join(ctx, flat, np.concatenate([rng.uniform(-10, 110, (40, 2)), [[50.0, 0.0], [1e6, 0.0]]]))
    # zero-width and zero-size boxes
    col = GeoArrowArray.points(np.stack([np.full(300, 2.5), rng.uniform(0, 10, 300)], 1))
    check_join(ctx, col, rng.uniform(-5, 15, (40, 2)))
    same = GeoArrowArray.points(np.full((50, 2), 1.25))
    _, nid, _, tied = check_join(ctx, same, rng.uniform(-5, 5, (20, 2)))
    assert (tied == 50).all() and (nid == 0).all()
    # 1e6 offsets with 1e-10 extents (far from the origin, tiny geometry)
    base = np.array([1e6, -2e6])
    tiny = [[tuple(base + rng.uniform(0, 1e-6, 2)), tuple(base + rng.uniform(0, 1e-6, 2))] for _ in range(300)]
    tl = GeoArrowArray.from_shapes(GeometryType.LINESTRING, tiny)
    check_join(ctx, tl, base + rng.uniform(-2e-6, 3e-6, (40, 2)))


def test_grid_cap(ctx):
    """>= 4.2 M right rows: G reaches the 2048 cap"""
    import torch

    n = 4_300_000
    xy = torch.empty((n, 2), dtype=torch.float64, device="cuda")
    engine.check(ctx.lib.gpl_gen_uniform_points(ctx._h, 9, 0, n, 1000.0, xy.data_ptr()))
    ctx.synchronize()
    host = xy.cpu().numpy()
    rhs = GeoArrowArray.points(host)
    rng = np.random.default_rng(2)
    P = np.concatenate([rng.uniform(-10, 1010, (24, 2)), host[:4] + 1e-9, [[5e5, 5e5]]])
    idx, nid, dist, tied = check_join(ctx, rhs, P)
    st = idx.stats()
    assert st["grid_cells_per_axis"] == 2048 and st["rows"] == n
    assert st["evaluations"] < 20 * len(P)


def test_bundled_datasets(ctx):
    from geopolars_b200 import datasets

    cities = datasets.read_dataset("naturalearth_cities").geometry.device.to_host()
    countries = datasets.read_dataset("naturalearth_lowres").geometry.device.to_host()
    nybb = datasets.read_dataset("nybb").geometry.device.to_host()
    assert cities.type == GeometryType.POINT
    check_join(ctx, countries, cities.xy, pvalid=cities.valid)
    lo, hi = nybb.xy.min(0), nybb.xy.max(0)
    rng = np.random.default_rng(4)
    check_join(ctx, nybb, lo + rng.uniform(-0.1, 1.1, (80, 2)) * (hi - lo))


def _referee_polys_batched(ctx, poly_xy, m, nv1, P, batch=100):
    """the referee for a POLYGON column of m one-ring polygons of nv1 coordinates each (device coordinates poly_xy):
    `distance` over batch x m rows per call (the points repeated, the polygons tiled)"""
    import torch

    dev = poly_xy.device
    tiled = poly_xy.repeat(batch, 1).contiguous()
    ro = torch.arange(batch * m + 1, dtype=torch.int64, device=dev) * nv1
    go = torch.arange(batch * m + 1, dtype=torch.int64, device=dev)
    rhs = ctx.wrap_device(GeometryType.POLYGON, batch * m, batch * m * nv1, tiled.data_ptr(), geom_off_ptr=go.data_ptr(), ring_off_ptr=ro.data_ptr(),
                          n_rings=batch * m, keepalive=(tiled, ro, go))
    nid, dist, tied = [], [], []
    for s in range(0, len(P), batch):
        Pb = P[s:s + batch]
        k = len(Pb)
        Pb = np.concatenate([Pb, np.repeat(Pb[-1:], batch - k, 0)])
        pt = torch.from_numpy(np.repeat(Pb, m, 0)).to(dev)
        col = ctx.wrap_device(GeometryType.POINT, batch * m, batch * m, pt.data_ptr(), keepalive=(pt,))
        torch.cuda.synchronize()  # the inputs were made on torch's stream, `distance` runs on the context's
        d = engine.distance(col, rhs)[0].reshape(batch, m)[:k]
        best = d.min(1)
        at = d == best[:, None]
        nid.append(np.argmax(at, 1)), dist.append(best), tied.append(at.sum(1))
    return np.concatenate(nid).astype(np.int32), np.concatenate(dist), np.concatenate(tied).astype(np.int32)


def test_ten_million_points_config2(ctx):
    """10 M uniform points x config 2's 10 k 64-vertex polygons"""
    import torch

    from geopolars_b200 import synth

    m, grid, cell, nv = 10_000, 100, 10.0, 64
    xy, ro, go = synth.star_polygons(m, grid, cell, nv)
    polys = ctx.upload(GeoArrowArray.polygons(xy, ro, go))
    n = 10_000_000
    pts = torch.empty((n, 2), dtype=torch.float64, device="cuda")
    engine.check(ctx.lib.gpl_gen_uniform_points(ctx._h, 2, 0, n, grid * cell, pts.data_ptr()))
    nid = torch.empty(n, dtype=torch.int32, device="cuda")
    dist = torch.empty(n, dtype=torch.float64, device="cuda")
    tied = torch.empty(n, dtype=torch.int32, device="cuda")
    idx = engine.NearestIndex(polys)
    idx.query_device(pts.data_ptr(), n, None, nid.data_ptr(), dist.data_ptr(), tied.data_ptr())
    ctx.synchronize()
    st = idx.stats()
    print("config2 10M stats", st)
    nid_h, dist_h, tied_h = nid.cpu().numpy(), dist.cpu().numpy(), tied.cpu().numpy()
    assert (nid_h >= 0).all() and (nid_h < m).all() and (tied_h >= 1).all() and st["overflow_points"] == 0
    # every point's distance is distance(point, rhs[nearest_id]) bit for bit (the rows gathered on the device)
    poly_t = torch.from_numpy(xy).cuda()
    nv1 = nv + 1
    for s in range(0, n, 2_500_000):
        e = min(n, s + 2_500_000)
        k = e - s
        g = poly_t.reshape(m, nv1, 2)[nid[s:e].to(torch.int64)].reshape(-1, 2).contiguous()
        gro = torch.arange(k + 1, dtype=torch.int64, device="cuda") * nv1
        ggo = torch.arange(k + 1, dtype=torch.int64, device="cuda")
        col = ctx.wrap_device(GeometryType.POLYGON, k, k * nv1, g.data_ptr(), geom_off_ptr=ggo.data_ptr(), ring_off_ptr=gro.data_ptr(), n_rings=k,
                              keepalive=(g, gro, ggo))
        pc = pts[s:e].contiguous()
        pcol = ctx.wrap_device(GeometryType.POINT, k, k, pc.data_ptr(), keepalive=(pc,))
        torch.cuda.synchronize()  # the gather ran on torch's stream, `distance` runs on the context's
        assert same_f64(engine.distance(pcol, col)[0], dist_h[s:e])
        del g, col
    # the contains join: a point inside polygon k has distance 0 and nearest_id k (config 2's polygons are disjoint)
    pip = engine.PipIndex(polys)
    first = torch.empty(n, dtype=torch.int32, device="cuda")
    pip.query_device(pts.data_ptr(), n, first.data_ptr())
    ctx.synchronize()
    first_h = first.cpu().numpy()
    inside = first_h >= 0
    assert inside.sum() > n // 10
    assert (nid_h[inside] == first_h[inside]).all() and (dist_h[inside] == 0).all() and (tied_h[inside] == 1).all()
    # a 20 k sample equals the referee
    P = pts.cpu().numpy()
    s = np.random.default_rng(8).choice(n, 20_000, replace=False)
    rn, rd, rt = _referee_polys_batched(ctx, poly_t, m, nv1, P[s])
    assert np.array_equal(nid_h[s], rn) and same_f64(dist_h[s], rd) and np.array_equal(tied_h[s], rt)
    # 2 000 of them against the independent CPU reference
    t = s[:2000]
    assert oracle_agrees(GeoArrowArray.polygons(xy, ro, go), P[t], None, INF, nid_h[t], dist_h[t]) > 1900


def test_accessor_and_guards(ctx):
    rng = np.random.default_rng(9)
    rows = shapes.random_rows(rng, "polygon", 100)
    rhs = GeoArrowArray.from_shapes(GeometryType.POLYGON, rows)
    P = np.concatenate([rng.uniform(-3, 13, (50, 2)), [[1e3, 1e3]]])
    pv = np.ones(len(P), bool)
    pv[3] = False
    lhs = GeoSeries(_device=ctx.upload(GeoArrowArray.points(P, valid=pv)))
    rs = GeoSeries(_device=ctx.upload(rhs))
    a, b, d = nearest_join(lhs, rs)
    idx = engine.NearestIndex(rs.device)
    nid, dist, tied = idx.query_array(lhs.device)
    assert len(a) == int(tied.sum()) and np.all(np.diff(a) >= 0)
    assert same_f64(d, dist[a]) and 3 not in a
    a2, b2, d2 = nearest_join(lhs, rs, how="left", max_distance=2.0)
    _, dist2, tied2 = idx.query_array(lhs.device, 2.0)
    miss = np.nonzero(tied2 == 0)[0]
    assert 3 in miss and len(miss) >= 1
    assert len(a2) == int(tied2.sum()) + len(miss) and sorted(set(a2.tolist())) == list(range(len(P)))
    assert (b2[np.isin(a2, miss)] == -1).all() and np.isnan(d2[np.isin(a2, miss)]).all()
    with pytest.raises(ValueError):
        nearest_join(lhs, rs, how="right")
    # left side must be Point
    with pytest.raises(_lib.MismatchedGeometry):
        idx.query_array(rs.device)
    # more than 2^31 - 1 points per call (checked before any access)
    import ctypes as C

    buf = np.zeros(8, np.int32)
    # max_distance = NaN as well: should the count check ever go, the argument check still rejects the call before any launch
    rc = ctx.lib.gpl_nearest_join(ctx._h, idx._h, C.c_void_p(1), (1 << 31), math.nan, C.c_void_p(buf.ctypes.data), None, None,
                                  engine.GPL_DEVICE)
    assert rc == -6
