"""Every pair list the library returns, read through gpl_pairs_copy / gpl_pairs_copy_distance directly (no host sort can hide
its order): sorted strictly by (lhs, rhs), the same bytes on a repeated call, the same set as a row-wise brute force over the
cross product, and NULL in *out when the call fails."""
import ctypes as C
import zlib

import numpy as np
import pytest
import torch

import shapes
from geopolars_b200 import GeoArrowArray, GeometryType, engine, synth

pytestmark = pytest.mark.gpu
GPL_ERR_UNSUPPORTED = -6

T = {
    "point": GeometryType.POINT,
    "multipoint": GeometryType.MULTIPOINT,
    "linestring": GeometryType.LINESTRING,
    "multilinestring": GeometryType.MULTILINESTRING,
    "polygon": GeometryType.POLYGON,
    "multipolygon": GeometryType.MULTIPOLYGON,
}
ARMS = [("polygon", "polygon"), ("multipolygon", "polygon"), ("polygon", "multipolygon"), ("point", "polygon"), ("polygon", "point"),
        ("point", "multipolygon"), ("linestring", "point"), ("point", "multilinestring"), ("multilinestring", "point"),
        ("linestring", "linestring"), ("multipolygon", "multipolygon"), ("multipoint", "polygon")]


def _read(ctx, h, with_distance=False):
    """(lhs, rhs[, dist]) of a pair list handle, straight from the library; frees it"""
    try:
        n = int(ctx.lib.gpl_pairs_count(h))
        lhs, rhs, dist = np.zeros(n, np.uint64), np.zeros(n, np.uint64), np.zeros(n, np.float64)
        if n:
            engine.check(ctx.lib.gpl_pairs_copy(ctx._h, h, lhs.ctypes.data, rhs.ctypes.data, engine.GPL_HOST))
            if with_distance:
                engine.check(ctx.lib.gpl_pairs_copy_distance(ctx._h, h, dist.ctypes.data, engine.GPL_HOST))
    finally:
        ctx.lib.gpl_pairs_free(h)
    return (lhs, rhs, dist) if with_distance else (lhs, rhs)


def _twice(ctx, call, with_distance=False):
    """run call(&h) twice: both lists strictly increasing in (lhs, rhs) and byte-identical; returns the first"""
    got = []
    for _ in range(2):
        h = C.c_void_p()
        engine.check(call(C.byref(h)))
        got.append(_read(ctx, h, with_distance))
    for u, v in zip(*got):
        assert u.tobytes() == v.tobytes()
    lhs, rhs = got[0][0], got[0][1]
    assert (lhs < (1 << 31)).all() and (rhs < (1 << 31)).all()
    key = (lhs << np.uint64(32)) | rhs
    assert (key[1:] > key[:-1]).all(), "not strictly increasing in (lhs, rhs)"
    return got[0]


def _stars(rng, n, span, rmin, rmax):
    return [[shapes.valid_star(rng, rng.uniform(0, span), rng.uniform(0, span), rng.uniform(rmin, rmax), int(rng.integers(3, 9)))]
            for _ in range(n)]


def _cross(ctx, ka, A, kb, B):
    """the two columns repeated over the cross product: row i * len(B) + j is (A[i], B[j])"""
    At = [a for a in A for _ in B]
    Bt = [b for _ in A for b in B]
    return ctx.upload(GeoArrowArray.from_shapes(T[ka], At)), ctx.upload(GeoArrowArray.from_shapes(T[kb], Bt))


def _pairs_of(hit, m):
    k = np.nonzero(hit)[0]
    return (k // m).astype(np.uint64), (k % m).astype(np.uint64)


@pytest.mark.parametrize("ka,kb", ARMS)
@pytest.mark.parametrize("predicate", ["intersects", "contains"])
def test_spatial_join_sorted_and_brute_force(ctx, ka, kb, predicate):
    rng = np.random.default_rng(zlib.crc32(f"pl{ka}x{kb}".encode()))
    n, m = 40, 33
    A = shapes.random_rows(rng, ka, n, span=12.0)
    B = shapes.random_rows(rng, kb, m, span=12.0)
    A = shapes.plant_touching(rng, ka, A, kb, (B * 2)[:n])
    if ka == "polygon" and kb == "polygon":
        for i in range(10):
            A[i], B[i] = [shapes.sq(2, 2, 8)], [shapes.valid_star(rng, 6, 6, 1.0, 5)]
    A[3] = None
    da, db = ctx.upload(GeoArrowArray.from_shapes(T[ka], A)), ctx.upload(GeoArrowArray.from_shapes(T[kb], B))
    p = engine.PREDICATES[predicate]
    lhs, rhs = _twice(ctx, lambda out: ctx.lib.gpl_spatial_join(ctx._h, da._h, db._h, p, out))
    # the dispatch of gpl_spatial_join, row-wise over every pair
    area, lines = ("polygon", "multipolygon"), ("linestring", "multilinestring")
    ta, tb = _cross(ctx, ka, A, kb, B)
    if ka == "point" and kb in area + lines:
        hit = engine.contains(tb, ta)
    elif kb == "point" and ka in area + lines:
        hit = engine.contains(ta, tb)
    elif ka in area and kb == "polygon":
        hit = engine.contains(ta, tb) if predicate == "contains" else engine.intersects(ta, tb)
    elif ka == "polygon" and kb == "multipolygon" and predicate == "intersects":
        hit = engine.intersects(ta, tb)
    else:
        hit = np.zeros(n * m, dtype=bool)
    want_l, want_r = _pairs_of(hit, m)
    assert np.array_equal(lhs, want_l) and np.array_equal(rhs, want_r)


def test_spatial_join_larger_repeat(ctx):
    """the 2 000 x 1 500 polygons of the general join's larger case: long cell lists, many hits per left row"""
    rng = np.random.default_rng(77)
    A, B = _stars(rng, 2000, 100, 0.5, 6), _stars(rng, 1500, 100, 0.3, 3)
    da, db = ctx.upload(GeoArrowArray.from_shapes(T["polygon"], A)), ctx.upload(GeoArrowArray.from_shapes(T["polygon"], B))
    for p in (0, 1):
        lhs, _ = _twice(ctx, lambda out: ctx.lib.gpl_spatial_join(ctx._h, da._h, db._h, p, out))
        assert len(lhs) > (500 if p == 0 else 20)


def test_overlay_joins_sorted_and_brute_force(ctx):
    rng = np.random.default_rng(2024)
    A, B = _stars(rng, 70, 30, 1.0, 5), _stars(rng, 60, 30, 0.5, 4)
    B[5] = A[7]  # an identical pair
    da, db = ctx.upload(GeoArrowArray.from_shapes(T["polygon"], A)), ctx.upload(GeoArrowArray.from_shapes(T["polygon"], B))
    lhs, rhs, area = _twice(ctx, lambda out: ctx.lib.gpl_overlay_area_join(ctx._h, da._h, db._h, out), with_distance=True)
    ta, tb = _cross(ctx, "polygon", A, "polygon", B)
    want_l, want_r = _pairs_of(engine.intersects(ta, tb), len(B))
    assert np.array_equal(lhs, want_l) and np.array_equal(rhs, want_r) and len(lhs) > 50
    want_area, _ = engine.intersection_area(ta, tb)
    assert want_area[(want_l * len(B) + want_r).astype(np.int64)].tobytes() == area.tobytes()
    # the geometry overlay join: a subset of those pairs, and the same pairs and geometry bytes twice
    got = []
    for _ in range(2):
        hp, ha = C.c_void_p(), C.c_void_p()
        engine.check(ctx.lib.gpl_overlay_join(ctx._h, da._h, db._h, C.byref(hp), C.byref(ha)))
        g = engine.DeviceArray(ctx, ha).to_host()
        got.append(_read(ctx, hp) + (g.xy, g.geom_off, g.part_off, g.ring_off))
    for u, v in zip(*got):
        assert np.asarray(u).tobytes() == np.asarray(v).tobytes()
    ol, orr = got[0][0], got[0][1]
    key = (ol << np.uint64(32)) | orr
    assert (key[1:] > key[:-1]).all() and 0 < len(key) and set(key.tolist()) <= set(((lhs << np.uint64(32)) | rhs).tolist())


def test_predicate_join_every_predicate_sorted(ctx):
    rng = np.random.default_rng(31)
    A = _stars(rng, 60, 25, 1.0, 5)
    B = _stars(rng, 50, 25, 0.5, 3) + [A[2], [shapes.sq(0, 0, 30)]]
    L = shapes.random_rows(rng, "linestring", 40, span=25.0)
    da, db = ctx.upload(GeoArrowArray.from_shapes(T["polygon"], A)), ctx.upload(GeoArrowArray.from_shapes(T["polygon"], B))
    dl = ctx.upload(GeoArrowArray.from_shapes(T["linestring"], L))
    codes = {k: v for k, v in engine.RELATE_PREDICATES.items() if k != "disjoint"}
    for lhs_col, rhs_col in ((da, db), (dl, da), (da, dl)):
        base, _ = _twice(ctx, lambda out: ctx.lib.gpl_predicate_join(ctx._h, lhs_col._h, rhs_col._h, 0, None, out))
        assert len(base) > 0
        for name, code in codes.items():
            pat = b"T*T***T**" if name == "relate_pattern" else None
            _twice(ctx, lambda out: ctx.lib.gpl_predicate_join(ctx._h, lhs_col._h, rhs_col._h, code, pat, out))


def test_points_in_polygons_nearest_dwithin_great_circle_sorted(ctx):
    rng = np.random.default_rng(5)
    xy, ro, go = synth.star_polygons(400, 20)
    polys = ctx.upload(GeoArrowArray.polygons(xy, ro, go))
    pts = ctx.upload(GeoArrowArray.points(synth.uniform_points(100_000, scale=200.0)))
    pip = engine.PipIndex(polys)
    _twice(ctx, lambda out: ctx.lib.gpl_contains_join_pairs_array(ctx._h, pip._h, pts._h, out))
    # nearest and distance-within, Point and LineString left sides (ties on a lattice)
    R = ctx.upload(GeoArrowArray.from_shapes(T["polygon"], _stars(rng, 400, 100, 0.5, 3)))
    lat = np.stack(np.meshgrid(np.arange(0, 100, 2.0), np.arange(0, 100, 2.0)), -1).reshape(-1, 2)
    lattice = ctx.upload(GeoArrowArray.points(lat))
    P = ctx.upload(GeoArrowArray.points(rng.uniform(0, 100, (20_000, 2))))
    Ls = ctx.upload(GeoArrowArray.from_shapes(T["linestring"], shapes.random_rows(rng, "linestring", 500, span=100.0)))
    ni = engine.NearestIndex(R)
    for left in (P, lattice):
        _twice(ctx, lambda out: ctx.lib.gpl_nearest_join_pairs_array(ctx._h, ni._h, left._h, float("inf"), out, None, engine.GPL_HOST))
    _twice(ctx, lambda out: ctx.lib.gpl_nearest_join_geom_pairs(ctx._h, ni._h, Ls._h, float("inf"), out, None, engine.GPL_HOST))
    for left in (P, Ls):
        for wd in (0, 1):
            _twice(ctx, lambda out: ctx.lib.gpl_dwithin_join_pairs(ctx._h, ni._h, left._h, 2.0, wd, out), with_distance=bool(wd))
    # great circle: (lon, lat) points
    gr = ctx.upload(GeoArrowArray.points(np.stack([rng.uniform(-180, 180, 5000), rng.uniform(-80, 80, 5000)], 1)))
    gl = ctx.upload(GeoArrowArray.points(np.stack([rng.uniform(-180, 180, 8000), rng.uniform(-80, 80, 8000)], 1)))
    gi = engine.GeoIndex(gr)
    for wd in (0, 1):
        _twice(ctx, lambda out: ctx.lib.gpl_geo_dwithin_join_pairs(ctx._h, gi._h, gl._h, 300e3, wd, out), with_distance=bool(wd))
    _twice(ctx, lambda out: ctx.lib.gpl_geo_nearest_join_pairs(ctx._h, gi._h, gl._h, float("inf"), out, None, engine.GPL_HOST))
    pip.free(), ni.free(), gi.free()


def test_error_leaves_out_null(ctx):
    """a call that fails stores NULL in *out (nothing to free, nothing leaked): 2^31 left rows are rejected before any access"""
    small = torch.zeros(16, dtype=torch.int64, device="cuda")
    p = small.data_ptr()
    big_poly = ctx.wrap_device(GeometryType.POLYGON, 1 << 31, 1 << 32, p, geom_off_ptr=p, ring_off_ptr=p, n_rings=1 << 31, keepalive=(small,))
    big_line = ctx.wrap_device(GeometryType.LINESTRING, 1 << 31, 1 << 32, p, geom_off_ptr=p, keepalive=(small,))
    rhs = ctx.upload(GeoArrowArray.from_shapes(T["polygon"], [[shapes.sq(0, 0, 1)], [shapes.sq(2, 2, 1)]]))

    def fails(call):
        h = C.c_void_p(0x1000)  # a stale value the call must overwrite
        assert call(C.byref(h)) == GPL_ERR_UNSUPPORTED
        assert h.value is None

    for p_ in (0, 1):
        fails(lambda out: ctx.lib.gpl_spatial_join(ctx._h, big_poly._h, rhs._h, p_, out))
    fails(lambda out: ctx.lib.gpl_overlay_area_join(ctx._h, big_poly._h, rhs._h, out))
    fails(lambda out: ctx.lib.gpl_predicate_join(ctx._h, big_poly._h, rhs._h, 0, None, out))
    ha = C.c_void_p(0x1000)
    fails(lambda out: ctx.lib.gpl_overlay_join(ctx._h, big_poly._h, rhs._h, out, C.byref(ha)))
    assert ha.value is None
    ni = engine.NearestIndex(rhs)
    fails(lambda out: ctx.lib.gpl_dwithin_join_pairs(ctx._h, ni._h, big_line._h, 1.0, 1, out))
    ni.free()
