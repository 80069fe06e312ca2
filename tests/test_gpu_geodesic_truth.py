"""The ellipsoid and sphere kernels on the GPU against the true geodesic (tests/golden/geodesic_truth.npz, 40-digit values
from tests/geodesic_truth.py): geodesic_length with Karney and Vincenty, haversine_distance and geodesic_length("haversine"),
geodesic_area signed and unsigned and the perimeter.  numpy only: the bounds (tests/geodesic_truth_bounds.py) are the ones
tests/test_geodesic_truth_cpu.py holds the CPU oracle to, set from its measured errors; the GPU maxima measured on an H100
are noted beside them."""
import numpy as np
import pytest

import geodesic_area_reference as R
from geopolars_b200 import GeoArrowArray, GeometryType, engine
from geodesic_truth_bounds import (
    HAVERSINE_K,
    KARNEY_BOUND_M,
    VINCENTY_BOUND_M,
    area_bound,
    err,
    haversine_bound,
    load,
    polygon_rows,
)

pytestmark = pytest.mark.gpu


def two_point_lines(pin):
    xy = pin.reshape(-1, 2)  # (lon1, lat1), (lon2, lat2) per pair
    return GeoArrowArray.linestrings(xy, np.arange(0, len(xy) + 1, 2, dtype=np.int64))


def test_karney_geodesic_length(ctx):
    """KARNEY_BOUND_M = 1e-8 m per segment (CPU oracle 6.3e-9 m; measured on an H100 80GB HBM3 at 700 W: 8.0e-9 m)"""
    fx = load()
    got, valid = engine.geodesic_length(ctx.upload(two_point_lines(fx["pair_in"])), "geodesic")
    assert valid.all()
    assert np.abs(err(got, fx["pair_s12"])).max() <= KARNEY_BOUND_M


def test_karney_multi_segment_rows(ctx):
    """rows that walk a fixture pair back and forth n times: within n segment bounds and n ulps of the sum of the truths"""
    fx = load()
    rng = np.random.default_rng(11)
    pick = rng.choice(len(fx["pair_in"]), 400, replace=False)
    n = rng.integers(1, 64, len(pick))
    xy, off = [], [0]
    for i, k in zip(pick, n):
        p = fx["pair_in"][i].reshape(2, 2)
        xy.append(np.concatenate([np.tile(p, (k // 2 + 1, 1))[: k + 1]]))
        off.append(off[-1] + k + 1)
    got, valid = engine.geodesic_length(ctx.upload(GeoArrowArray.linestrings(np.concatenate(xy), np.array(off))), "geodesic")
    truth = fx["pair_s12"][pick]
    want = n * truth[:, 0] + n * truth[:, 1]
    assert valid.all()
    assert np.all(np.abs(got - want) <= n * KARNEY_BOUND_M + n * np.spacing(want))


def test_vincenty_geodesic_length(ctx, og, conv):
    """VINCENTY_BOUND_M = 2e-4 m where it converges (CPU oracle 7.9e-5 m, H100 7.9e-5 m); null exactly where the
    oracle is"""
    fx = load()
    arr = two_point_lines(fx["pair_in"])
    got, valid = engine.geodesic_length(ctx.upload(arr), "vincenty")
    want = og.geodesic_length(conv(arr), "vincenty", threads=0)
    assert np.array_equal(valid, ~np.isnan(want)) and valid.sum() > 2000
    assert np.abs(err(got[valid], fx["pair_s12"][valid])).max() <= VINCENTY_BOUND_M


def test_haversine(ctx, og):
    """|dd| <= K eps R (1 + (|lon1| + |lon2|) / 180 + 1 / sqrt(1 - a)), HAVERSINE_K = 4 (CPU oracle 2.0, H100
    1.7, both on pairs under 100 m), for the row-wise op and the length; NaN (geo's unclamped asin of a rounded above 1) exactly where
    the oracle gives it"""
    fx = load()
    pin = fx["pair_in"]
    bound = haversine_bound(*pin.T)
    want = np.array([og.geodesic_distance("haversine", *p) for p in pin])
    d, v = engine.haversine_distance(ctx.upload(GeoArrowArray.points(pin[:, :2].copy())), ctx.upload(GeoArrowArray.points(pin[:, 2:].copy())))
    g, gv = engine.geodesic_length(ctx.upload(two_point_lines(pin)), "haversine")
    for got, ok in ((d, v), (g, gv)):
        assert ok.all()
        fin = ~np.isnan(got)
        assert np.array_equal(fin, ~np.isnan(want))
        assert np.all(np.abs(err(got[fin], fx["pair_haversine"][fin])) <= bound[fin])


@pytest.mark.parametrize("signed", [True, False])
def test_geodesic_area_and_perimeter(ctx, signed):
    """area within AREA_K = 16 eps (scale + |A|), unsigned (scale + rings area0) (CPU reference 10.5 and 1.0, H100 10.5 and
    3.1); perimeter within KARNEY_BOUND_M per edge (H100 3.1e-9 m)"""
    fx = load()
    rows = polygon_rows(fx)
    key = "poly_area_signed" if signed else "poly_area_unsigned"
    edges = np.diff(fx["poly_edge_off"][fx["poly_part_off"][fx["poly_row_off"]]])
    for multi, gt, kind in ((False, GeometryType.POLYGON, "polygon"), (True, GeometryType.MULTIPOLYGON, "multipolygon")):
        sel = np.flatnonzero(fx["poly_multi"] == multi)
        shapes = [rows[i] for i in sel]
        a, p, v = engine.geodesic_area(ctx.upload(GeoArrowArray.from_shapes(gt, shapes)), signed)
        scale = R.geodesic_area(shapes, kind, signed)[3]
        assert v.all()
        assert np.all(np.abs(err(a, fx[key][sel])) <= area_bound(fx, sel, scale, signed))
        assert np.all(np.abs(err(p, fx["poly_perimeter"][sel])) <= KARNEY_BOUND_M * edges[sel])
