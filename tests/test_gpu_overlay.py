"""Intersection area and the area-weighted overlay join (DESIGN.md §4.16) on the GPU: row-wise values against the exact
cut-and-classify referee, self-area and symmetry on the bundled datasets, partition identities at scale, the join's row
set against the oracle's row-wise intersects over full cross products, and determinism."""
import numpy as np
import pytest

import nearest_reference as nr
import overlay_reference as ref
import shapes
from geopolars_b200 import GeoArrowArray, GeometryType, _lib, datasets, engine, synth
from geopolars_b200.geoseries import GeoSeries, overlay_area_join
from test_gpu_nearest_geom import to_og
from test_overlay_area_model import case_pairs, known_cases

P, MP = GeometryType.POLYGON, GeometryType.MULTIPOLYGON


def tol(a, b):
    """1e-9 (area(a) + area(b)) + 1e-12 L², L the diagonal of the union of the two envelopes"""
    pts = np.array([p for m in (a, b) for rings in m for r in rings for p in r], dtype=np.float64).reshape(-1, 2)
    diag = float(np.hypot(*(pts.max(0) - pts.min(0)))) if len(pts) else 0.0
    return 1e-9 * float(ref.polygon_area(a) + ref.polygon_area(b)) + 1e-12 * diag * diag


def upload(ctx, t, rows):
    return ctx.upload(GeoArrowArray.from_shapes(t, rows))


def gather(a: GeoArrowArray, idx) -> GeoArrowArray:
    t = nr.take(to_og(a), np.asarray(idx, dtype=np.int64))
    return GeoArrowArray(a.type, t.xy, geom_off=t.geom_off, part_off=t.part_off, ring_off=t.ring_off)


@pytest.mark.gpu
def test_rowwise_against_the_exact_referee(ctx, og):
    pairs = case_pairs() + [(a, b) for a, b, _ in known_cases() if a and b]
    A, B = [a for a, _ in pairs], [b for _, b in pairs]
    got, valid = engine.intersection_area(upload(ctx, MP, A), upload(ctx, MP, B))
    assert valid.all()
    closures_meet = og.intersects_rowwise(to_og(GeoArrowArray.from_shapes(MP, A)), to_og(GeoArrowArray.from_shapes(MP, B)))
    for i, (a, b) in enumerate(pairs):
        want = ref.intersection_area(a, b)
        assert got[i] >= 0.0 and abs(got[i] - float(want)) <= tol(a, b), (i, a, b, got[i], want)
        if not closures_meet[i]:
            assert got[i] == 0.0, (i, got[i])
    # the same rows as Polygon columns (single-member rows) in all four type combinations: the same bits
    single = [i for i, (a, b) in enumerate(pairs) if len(a) == 1 and len(b) == 1]
    pa = upload(ctx, P, [pairs[i][0][0] for i in single])
    pb = upload(ctx, P, [pairs[i][1][0] for i in single])
    ma = upload(ctx, MP, [pairs[i][0] for i in single])
    mb = upload(ctx, MP, [pairs[i][1] for i in single])
    for x, y in ((pa, pb), (pa, mb), (ma, pb), (ma, mb)):
        v, ok = engine.intersection_area(x, y)
        assert ok.all() and np.array_equal(v.view(np.uint64), got[single].view(np.uint64))


@pytest.mark.gpu
def test_known_answers_and_symmetry(ctx):
    cases = [c for c in known_cases() if c[0] and c[1]]
    a = upload(ctx, MP, [c[0] for c in cases])
    b = upload(ctx, MP, [c[1] for c in cases])
    v, ok = engine.intersection_area(a, b)
    w, ok2 = engine.intersection_area(b, a)
    assert ok.all() and ok2.all()
    for i, (x, y, want) in enumerate(cases):
        assert abs(v[i] - float(want)) <= tol(x, y) and abs(w[i] - float(want)) <= tol(x, y), (x, y, v[i], w[i])
    sq = shapes.sq
    v, _ = engine.intersection_area(upload(ctx, P, [[sq(0, 0, 2)], [sq(0, 0, 1)]]), upload(ctx, P, [[sq(1, 1, 2)], [sq(5, 5, 1)]]))
    assert v.tolist() == [1.0, 0.0]


@pytest.mark.gpu
def test_nulls_empties_nonfinite_and_errors(ctx):
    sq = shapes.sq
    A = [[sq(0, 0, 2)], None, [], [sq(0, 0, 2)], [[(0, 0), (np.nan, 0), (1, 1), (0, 0)]], [sq(0, 0, 2)], [sq(0, 0, 2)]]
    B = [[sq(1, 1, 2)], [sq(0, 0, 1)], [sq(0, 0, 1)], None, [sq(0, 0, 1)], [], [[(0, 0), (1, 0), (np.inf, 1), (0, 0)]]]
    v, ok = engine.intersection_area(upload(ctx, P, A), upload(ctx, P, B))
    assert ok.tolist() == [True, False, True, False, False, True, False]
    assert v[0] == 1.0 and v[2] == 0.0 and v[5] == 0.0 and np.isnan(v[[1, 3, 4, 6]]).all()
    s = GeoSeries(_device=upload(ctx, P, A)).geo.intersection_area(GeoSeries(_device=upload(ctx, P, B)))
    assert s.null_count == 4 and s[0].as_py() == 1.0
    pts = ctx.upload(GeoArrowArray.from_shapes(GeometryType.POINT, [(0, 0)] * len(A)))
    lines = ctx.upload(GeoArrowArray.from_shapes(GeometryType.LINESTRING, [[(0, 0), (1, 1)]] * len(A)))
    for bad in (pts, lines):
        with pytest.raises(_lib.MismatchedGeometry, match=r"Expected \(Multi\)Polygon x \(Multi\)Polygon"):
            engine.intersection_area(upload(ctx, P, A), bad)
        with pytest.raises(_lib.MismatchedGeometry, match=r"Expected \(Multi\)Polygon x \(Multi\)Polygon"):
            engine.overlay_area_join(bad, upload(ctx, P, A))
    with pytest.raises(_lib.ShapeError):
        engine.intersection_area(upload(ctx, P, A), upload(ctx, P, B[:3]))


def dataset(name):
    return datasets.read_dataset(name).geometry.device


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["nybb", "naturalearth_lowres"])
def test_self_area_and_symmetry_on_datasets(ctx, name):
    d = dataset(name)
    host = d.to_host()
    area = np.abs(engine.area(d))
    v, ok = engine.intersection_area(d, d)
    assert ok.all()
    assert np.all(np.abs(v - area) <= 1e-9 * area), np.max(np.abs(v - area) / area)
    # symmetry: each row against the next one (neighbours share borders)
    nxt = ctx.upload(gather(host, (np.arange(len(host)) + 1) % len(host)))
    ab, _ = engine.intersection_area(d, nxt)
    ba, _ = engine.intersection_area(nxt, d)
    scale = area + np.roll(area, -1)
    assert np.all(np.abs(ab - ba) <= 1e-9 * scale)


def square_grid(x0, y0, step, nx, ny):
    xs = x0 + step * np.arange(nx + 1)
    ys = y0 + step * np.arange(ny + 1)
    rows = []
    for j in range(ny):
        for i in range(nx):
            a, b, c, d = float(xs[i]), float(ys[j]), float(xs[i + 1]), float(ys[j + 1])
            rows.append([[(a, b), (c, b), (c, d), (a, d), (a, b)]])
    return rows


def check_partition(ctx, lhs, grid_rows, rel=1e-9):
    rhs = upload(ctx, P, grid_rows)
    a, b, area = engine.overlay_area_join(lhs, rhs)
    assert np.all(area >= 0.0)
    want = np.abs(engine.area(lhs))
    sums = np.bincount(a.astype(np.int64), weights=area, minlength=len(lhs))
    assert np.all(np.abs(sums - want) <= rel * want), np.max(np.abs(sums - want) / want)
    return a, b, area


@pytest.mark.gpu
def test_partition_identity_at_scale(ctx):
    check_partition(ctx, dataset("naturalearth_lowres"), square_grid(-180.0, -90.0, 5.0, 72, 36))
    xy, ring_off, geom_off = synth.star_polygons()
    stars = ctx.upload(GeoArrowArray(P, xy, geom_off=geom_off, ring_off=ring_off))
    a, _, _ = check_partition(ctx, stars, square_grid(0.0, 0.0, 5.0, 200, 200))
    assert len(np.unique(a)) == 10_000
    nybb = dataset("nybb")
    box = engine.bounds(nybb)
    x0, y0 = float(np.floor(box[:, 0].min())), float(np.floor(box[:, 1].min()))
    step = 4000.0
    nx, ny = int(np.ceil((box[:, 2].max() - x0) / step)), int(np.ceil((box[:, 3].max() - y0) / step))
    check_partition(ctx, nybb, square_grid(x0, y0, step, nx, ny))


COMBOS = [(P, P), (P, MP), (MP, P), (MP, MP)]


@pytest.mark.gpu
@pytest.mark.parametrize("tl,tr", COMBOS)
def test_join_rows_and_bits_against_the_cross_product(ctx, og, tl, tr):
    rng = np.random.default_rng(7 + int(tl) * 10 + int(tr))
    kind = {P: "polygon", MP: "multipolygon"}
    L = GeoArrowArray.from_shapes(tl, shapes.random_rows(rng, kind[tl], 300) + [None])
    R = GeoArrowArray.from_shapes(tr, shapes.random_rows(rng, kind[tr], 300) + [None])
    ld, rd = ctx.upload(L), ctx.upload(R)
    a, b, area = engine.overlay_area_join(ld, rd)
    ii, jj = np.meshgrid(np.arange(len(L)), np.arange(len(R)), indexing="ij")
    ii, jj = ii.ravel(), jj.ravel()
    hit = og.intersects_rowwise(to_og(gather(L, ii)), to_og(gather(R, jj)))
    want = set(zip(ii[hit].tolist(), jj[hit].tolist()))
    assert len(want) > 100
    assert set(zip(a.tolist(), b.tolist())) == want and len(a) == len(want)
    assert np.all(np.lexsort((b, a)) == np.arange(len(a)))
    # the area of each pair: bit for bit the row-wise value on the gathered rows
    v, ok = engine.intersection_area(ctx.upload(gather(L, a)), ctx.upload(gather(R, b)))
    assert ok.all() and np.array_equal(v.view(np.uint64), area.view(np.uint64))
    # how="left" adds exactly the unmatched left rows once, with rhs -1 and NaN
    la, lb, ld_ = overlay_area_join(GeoSeries(_device=ld), GeoSeries(_device=rd), how="left")
    miss = sorted(set(range(len(L))) - set(a.tolist()))
    assert len(la) == len(a) + len(miss)
    extra = lb == -1
    assert la[extra].tolist() == miss and np.isnan(ld_[extra]).all()
    assert np.array_equal(ld_[~extra].view(np.uint64), area.view(np.uint64))
    # determinism
    a2, b2, area2 = engine.overlay_area_join(ld, rd)
    assert np.array_equal(a, a2) and np.array_equal(b, b2) and np.array_equal(area.view(np.uint64), area2.view(np.uint64))
    v2, _ = engine.intersection_area(ctx.upload(gather(L, a)), ctx.upload(gather(R, b)))
    assert np.array_equal(v.view(np.uint64), v2.view(np.uint64))


@pytest.mark.gpu
def test_join_empty_sides_and_touching_pairs(ctx):
    sq = shapes.sq
    a, b, area = engine.overlay_area_join(upload(ctx, P, [[sq(0, 0, 1)]]), upload(ctx, P, [[sq(1, 0, 1)], [sq(5, 5, 1)], [sq(0, 0, 1)]]))
    assert a.tolist() == [0, 0] and b.tolist() == [0, 2] and area.tolist() == [0.0, 1.0]
    a, b, area = engine.overlay_area_join(upload(ctx, P, []), upload(ctx, P, [[sq(0, 0, 1)]]))
    assert len(a) == len(b) == len(area) == 0
