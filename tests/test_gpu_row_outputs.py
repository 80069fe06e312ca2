"""Row results written to device memory (GPL_DEVICE) are byte-identical to the same results copied to the host (GPL_HOST),
values and validity bitmap alike, and every entry point that takes `mem` rejects any other value before it launches or
copies anything."""
import ctypes as C

import numpy as np
import pytest

import shapes
from geopolars_b200 import GeoArrowArray, GeometryType
from geopolars_b200._lib import check

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

HOST, DEVICE, BAD = 0, 1, 2
INVALID_ARG = -7
TYPES = {"point": GeometryType.POINT, "multipoint": GeometryType.MULTIPOINT, "linestring": GeometryType.LINESTRING,
         "multilinestring": GeometryType.MULTILINESTRING, "polygon": GeometryType.POLYGON, "multipolygon": GeometryType.MULTIPOLYGON}
N = 300


def column(kind, seed, n=N):
    """n seeded rows of `kind` with a null row every 7 rows and an empty row every 11"""
    rows = shapes.random_rows(np.random.default_rng(seed), kind, n)
    for i in range(0, n, 11):
        rows[i] = (np.nan, np.nan) if kind == "point" else []
    for i in range(3, n, 7):
        rows[i] = None
    return GeoArrowArray.from_shapes(TYPES[kind], rows)


_cache = {}


def dev(ctx, kind, seed):
    key = (kind, seed)
    if key not in _cache:
        _cache[key] = ctx.upload(column(kind, seed))
    return _cache[key]


def run_both(ctx, call, outs):
    """call(mem, *ptrs) with outs = [(dtype, count, nullable)]: the GPL_HOST results and the GPL_DEVICE results (in torch
    device buffers), once with every output and once with the nullable outputs NULL"""
    for drop in (False, True):
        keep = [not (drop and nullable) for _, _, nullable in outs]
        if drop and all(keep):
            continue
        host = [np.full(np.dtype(dt).itemsize * k, 0x5A, dtype=np.uint8).view(dt) if kp else None for (dt, k, _), kp in zip(outs, keep)]
        check(call(HOST, *[None if h is None else C.c_void_p(h.ctypes.data) for h in host]))
        devb = [torch.full((np.dtype(dt).itemsize * k,), 0x5A, dtype=torch.uint8, device="cuda") if kp else None
                for (dt, k, _), kp in zip(outs, keep)]
        torch.cuda.synchronize()
        check(call(DEVICE, *[None if d is None else C.c_void_p(d.data_ptr()) for d in devb]))
        ctx.synchronize()
        for h, d in zip(host, devb):
            if h is None:
                continue
            assert h.view(np.uint8).tobytes() == d.cpu().numpy().tobytes()


def bitmap(n):
    return (np.uint8, (n + 7) // 8, True)


def bitmap_out(n):
    return (np.uint8, (n + 7) // 8, False)


@pytest.mark.parametrize("kind", list(TYPES))
def test_unary_rows(ctx, kind):
    lib, cx = ctx.lib, ctx._h
    a = dev(ctx, kind, 1)
    h = a._h
    run_both(ctx, lambda m, o: lib.gpl_area(cx, h, o, m), [(np.float64, N, False)])
    run_both(ctx, lambda m, o: lib.gpl_euclidean_length(cx, h, o, m), [(np.float64, N, False)])
    run_both(ctx, lambda m, o: lib.gpl_geom_type(cx, h, o, m), [(np.int8, N, False)])
    run_both(ctx, lambda m, o: lib.gpl_is_empty(cx, h, o, m), [bitmap_out(N)])
    run_both(ctx, lambda m, o: lib.gpl_is_ring(cx, h, o, m), [bitmap_out(N)])
    run_both(ctx, lambda m, o: lib.gpl_envelope(cx, h, None, o, m), [(np.float64, 4 * N, False)])
    for mode in (0, 1):
        run_both(ctx, lambda m, o: lib.gpl_envelope_query(cx, h, 2.0, 2.0, 8.0, 8.0, mode, o, m), [bitmap_out(N)])
    for method in (0, 1, 2):
        run_both(ctx, lambda m, o, v: lib.gpl_geodesic_length(cx, h, method, o, v, m), [(np.float64, N, False), bitmap(N)])
    for sign in (0, 1):
        run_both(ctx, lambda m, ar, pe, v: lib.gpl_geodesic_area(cx, h, sign, ar, pe, v, m),
                 [(np.float64, N, True), (np.float64, N, False), bitmap(N)])
        run_both(ctx, lambda m, ar, v: lib.gpl_geodesic_area(cx, h, sign, ar, None, v, m), [(np.float64, N, False), bitmap(N)])
    run_both(ctx, lambda m, o, v: lib.gpl_is_valid(cx, h, o, v, m), [(np.int8, N, False), bitmap(N)])
    if kind == "point":
        run_both(ctx, lambda m, o: lib.gpl_x(cx, h, o, m), [(np.float64, N, False)])
        run_both(ctx, lambda m, o: lib.gpl_y(cx, h, o, m), [(np.float64, N, False)])
        b = dev(ctx, "point", 2)._h
        run_both(ctx, lambda m, o, v: lib.gpl_haversine_distance(cx, h, b, o, v, m), [(np.float64, N, False), bitmap(N)])


@pytest.mark.parametrize("ka", list(TYPES))
@pytest.mark.parametrize("kb", list(TYPES))
def test_binary_rows(ctx, ka, kb):
    lib, cx = ctx.lib, ctx._h
    a, b = dev(ctx, ka, 3)._h, dev(ctx, kb, 4)._h
    run_both(ctx, lambda m, o, v: lib.gpl_distance(cx, a, b, o, v, m), [(np.float64, N, False), bitmap(N)])
    run_both(ctx, lambda m, o: lib.gpl_intersects(cx, a, b, o, m), [bitmap_out(N)])
    run_both(ctx, lambda m, o, v: lib.gpl_relate(cx, a, b, o, v, m), [(np.int8, 9 * N, False), bitmap(N)])
    for pred in (0, 2, 5, 9):
        run_both(ctx, lambda m, o: lib.gpl_relate_predicate(cx, a, b, pred, None, o, m), [bitmap_out(N)])
    area_a, area_b = ka in ("polygon", "multipolygon"), kb in ("polygon", "multipolygon")
    if kb == "point" and ka in ("linestring", "multilinestring", "polygon", "multipolygon"):
        run_both(ctx, lambda m, o: lib.gpl_contains(cx, a, b, o, m), [bitmap_out(N)])
    if area_a and kb == "polygon":
        run_both(ctx, lambda m, o: lib.gpl_contains_polygon(cx, a, b, o, m), [bitmap_out(N)])
    if area_a and area_b:
        run_both(ctx, lambda m, o, v: lib.gpl_intersection_area(cx, a, b, o, v, m), [(np.float64, N, False), bitmap(N)])
    if ka in ("linestring", "multilinestring") and area_b:
        run_both(ctx, lambda m, o, v: lib.gpl_clip_length(cx, a, b, o, v, m), [(np.float64, N, False), bitmap(N)])


@pytest.mark.parametrize("kind", list(TYPES))
def test_dwithin_counts(ctx, kind):
    lib, cx = ctx.lib, ctx._h
    idx = C.c_void_p()
    check(lib.gpl_nearest_index_build(cx, dev(ctx, "polygon", 5)._h, C.byref(idx)))
    try:
        h = dev(ctx, kind, 6)._h
        run_both(ctx, lambda m, o: lib.gpl_dwithin_count(cx, idx, h, 0.5, o, m), [(np.int32, N, False)])
    finally:
        lib.gpl_nearest_index_free(idx)
    gidx = C.c_void_p()
    check(lib.gpl_geo_index_build(cx, dev(ctx, "point", 7)._h, C.byref(gidx)))
    try:
        h = dev(ctx, "point", 8)._h
        run_both(ctx, lambda m, o: lib.gpl_geo_dwithin_count(cx, gidx, h, 100_000.0, o, m), [(np.int32, N, False)])
    finally:
        lib.gpl_geo_index_free(gidx)


def test_unknown_mem_is_rejected_before_any_work(ctx):
    lib, cx = ctx.lib, ctx._h
    z = {k: ctx.upload(column(k, 9, 0)) for k in ("point", "linestring", "polygon", "multipolygon")}
    pt, ls, pg, mp = (z[k]._h for k in ("point", "linestring", "polygon", "multipolygon"))
    bufs = [torch.zeros(64, dtype=torch.int64, device="cuda") for _ in range(6)]
    torch.cuda.synchronize()
    p = [C.c_void_p(b.data_ptr()) for b in bufs]
    n_bytes = C.c_int64(0)
    n_pairs = C.c_int64(0)
    pip, nidx, gidx = C.c_void_p(), C.c_void_p(), C.c_void_p()
    few, few_pts = ctx.upload(column("polygon", 10, 20)), ctx.upload(column("point", 11, 20))
    check(lib.gpl_pip_index_build(cx, few._h, C.byref(pip)))
    check(lib.gpl_nearest_index_build(cx, few._h, C.byref(nidx)))
    check(lib.gpl_geo_index_build(cx, few_pts._h, C.byref(gidx)))
    pairs, dpairs = C.c_void_p(), C.c_void_p()
    check(lib.gpl_spatial_join(cx, pg, pg, 0, C.byref(pairs)))
    check(lib.gpl_dwithin_join_pairs(cx, nidx, pt, 1.0, 1, C.byref(dpairs)))
    out = C.c_void_p()
    calls = {
        "gpl_array_copy_out": lambda m: lib.gpl_array_copy_out(cx, pg, p[0], p[1], p[2], p[3], p[4], m),
        "gpl_wkb_decode": lambda m: lib.gpl_wkb_decode(cx, p[0], p[1], 64, p[2], 0, m, C.byref(out)),
        "gpl_wkb_encode": lambda m: lib.gpl_wkb_encode(cx, pg, p[0], 64, p[1], C.byref(n_bytes), m),
        "gpl_area": lambda m: lib.gpl_area(cx, pg, p[0], m),
        "gpl_envelope": lambda m: lib.gpl_envelope(cx, pg, None, p[0], m),
        "gpl_euclidean_length": lambda m: lib.gpl_euclidean_length(cx, ls, p[0], m),
        "gpl_geodesic_length": lambda m: lib.gpl_geodesic_length(cx, ls, 0, p[0], p[1], m),
        "gpl_geodesic_area": lambda m: lib.gpl_geodesic_area(cx, pg, 0, p[0], p[1], p[2], m),
        "gpl_distance": lambda m: lib.gpl_distance(cx, pg, pg, p[0], p[1], m),
        "gpl_intersects": lambda m: lib.gpl_intersects(cx, pg, pg, p[0], m),
        "gpl_contains": lambda m: lib.gpl_contains(cx, pg, pt, p[0], m),
        "gpl_geom_type": lambda m: lib.gpl_geom_type(cx, pg, p[0], m),
        "gpl_is_empty": lambda m: lib.gpl_is_empty(cx, pg, p[0], m),
        "gpl_is_ring": lambda m: lib.gpl_is_ring(cx, ls, p[0], m),
        "gpl_x": lambda m: lib.gpl_x(cx, pt, p[0], m),
        "gpl_y": lambda m: lib.gpl_y(cx, pt, p[0], m),
        "gpl_contains_polygon": lambda m: lib.gpl_contains_polygon(cx, mp, pg, p[0], m),
        "gpl_relate": lambda m: lib.gpl_relate(cx, pg, pg, p[0], p[1], m),
        "gpl_relate_predicate": lambda m: lib.gpl_relate_predicate(cx, pg, pg, 0, None, p[0], m),
        "gpl_pairs_copy": lambda m: lib.gpl_pairs_copy(cx, pairs, p[0], p[1], m),
        "gpl_pairs_copy_distance": lambda m: lib.gpl_pairs_copy_distance(cx, dpairs, p[0], m),
        "gpl_envelope_query": lambda m: lib.gpl_envelope_query(cx, pg, 0.0, 0.0, 1.0, 1.0, 0, p[0], m),
        "gpl_contains_join": lambda m: lib.gpl_contains_join(cx, pip, p[0], 0, p[1], p[2], m),
        "gpl_contains_join_counts": lambda m: lib.gpl_contains_join_counts(cx, pip, p[0], 0, p[1], p[2], m),
        "gpl_contains_join_array": lambda m: lib.gpl_contains_join_array(cx, pip, pt, p[0], p[1], m),
        "gpl_contains_join_pairs": lambda m: lib.gpl_contains_join_pairs(cx, pip, p[0], 0, p[1], p[2], C.byref(n_pairs), m),
        "gpl_join_histogram": lambda m: lib.gpl_join_histogram(cx, p[0], 0, p[1], 20, m),
        "gpl_nearest_join": lambda m: lib.gpl_nearest_join(cx, nidx, p[0], 0, float("inf"), p[1], p[2], p[3], m),
        "gpl_nearest_join_array": lambda m: lib.gpl_nearest_join_array(cx, nidx, pt, float("inf"), p[0], p[1], p[2], m),
        "gpl_nearest_join_pairs_array": lambda m: lib.gpl_nearest_join_pairs_array(cx, nidx, pt, float("inf"), C.byref(out), p[0], m),
        "gpl_nearest_join_geom": lambda m: lib.gpl_nearest_join_geom(cx, nidx, ls, float("inf"), p[0], p[1], p[2], m),
        "gpl_nearest_join_geom_pairs": lambda m: lib.gpl_nearest_join_geom_pairs(cx, nidx, ls, float("inf"), C.byref(out), p[0], m),
        "gpl_dwithin_count": lambda m: lib.gpl_dwithin_count(cx, nidx, pt, 1.0, p[0], m),
        "gpl_intersection_area": lambda m: lib.gpl_intersection_area(cx, pg, pg, p[0], p[1], m),
        "gpl_is_valid": lambda m: lib.gpl_is_valid(cx, pg, p[0], p[1], m),
        "gpl_dissolve": lambda m: lib.gpl_dissolve(cx, pg, p[0], m, 1, C.byref(out)),
        "gpl_clip_length": lambda m: lib.gpl_clip_length(cx, ls, pg, p[0], p[1], m),
        "gpl_haversine_distance": lambda m: lib.gpl_haversine_distance(cx, pt, pt, p[0], p[1], m),
        "gpl_geo_dwithin_count": lambda m: lib.gpl_geo_dwithin_count(cx, gidx, pt, 1.0, p[0], m),
        "gpl_geo_nearest_join": lambda m: lib.gpl_geo_nearest_join(cx, gidx, pt, float("inf"), p[0], p[1], p[2], m),
        "gpl_geo_nearest_join_pairs": lambda m: lib.gpl_geo_nearest_join_pairs(cx, gidx, pt, float("inf"), C.byref(out), p[0], m),
    }
    try:
        for name, call in calls.items():
            before = ctx.launch_count
            rc = call(BAD)
            assert rc == INVALID_ARG, (name, rc)
            assert b"mem" in lib.gpl_last_error(), name
            assert ctx.launch_count == before, name
        ctx.synchronize()
        assert all(int(b.abs().sum()) == 0 for b in bufs)  # nothing was written to any output
    finally:
        lib.gpl_pairs_free(pairs)
        lib.gpl_pairs_free(dpairs)
        lib.gpl_pip_index_free(pip)
        lib.gpl_nearest_index_free(nidx)
        lib.gpl_geo_index_free(gidx)
