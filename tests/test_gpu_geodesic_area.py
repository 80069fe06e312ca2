"""Geodesic area and perimeter on WGS84 (gpl_geodesic_area, DESIGN.md §4.17) on the GPU: closed forms, random polygons and
multipolygons against the CPU reference (tests/geodesic_area_reference.py), nulls and other types, the bundled datasets,
determinism and the multi-pass path."""
import math

import numpy as np
import pytest

import geodesic_area_reference as R
from geopolars_b200 import GeoArrowArray, GeometryType, datasets, engine

pytestmark = pytest.mark.gpu

P, MP = GeometryType.POLYGON, GeometryType.MULTIPOLYGON
QUARTER_MERIDIAN = 10001965.729


def run(ctx, arr, signed=True):
    return engine.geodesic_area(ctx.upload(arr), signed)


def rel(a, b):
    return abs(a - b) / max(abs(a), abs(b), 1e-300)


def assert_matches(got, want):
    """|d area| <= 1e-9 |A| + 1e-14 scale (the summed magnitudes of the terms of every S12, geodesic_area_reference), perimeter
    1e-9 relative, identical validity"""
    a, p, v = got
    wa, wp, wv, scale = want
    assert np.array_equal(v, wv)
    assert np.all(np.abs(a[v] - wa[v]) <= 1e-9 * np.abs(wa[v]) + 1e-14 * scale[v])
    assert np.all(np.abs(p[v] - wp[v]) <= 1e-9 * np.abs(wp[v]))
    assert np.isnan(a[~v]).all() and np.isnan(p[~v]).all()


def test_closed_forms(ctx):
    rows, want = [], []
    for dlam in (1, 45, 90, 135):
        tri = [(0.0, 0.0), (dlam, 0.0), (0.0, 90.0)]
        a = R.AREA0 * dlam / 720
        rows += [[tri], [list(reversed(tri))], [[(0.0, 0.0), (0.0, -90.0), (dlam, 0.0)]]]
        want += [(a, R.A * dlam * math.pi / 180 + 2 * QUARTER_MERIDIAN), (-a, None), (a, None)]
    arr = GeoArrowArray.from_shapes(P, rows)
    sa, sp, sv = run(ctx, arr, True)
    ua, up, uv = run(ctx, arr, False)
    assert sv.all() and uv.all() and np.array_equal(sp, up)
    for i, (ws, wper) in enumerate(want):
        assert rel(sa[i], ws) < 1e-12
        assert rel(ua[i], ws if ws > 0 else R.AREA0 + ws) < 1e-12
        if wper is not None:
            assert abs(sp[i] - wper) < 1e-3
    # published geographiclib values and the pole ring both ways
    polar = [(0, 89), (90, 89), (180, 89), (270, 89)]
    arr = GeoArrowArray.from_shapes(P, [[polar], [list(reversed(polar))], [[(-1, 0), (0, -1), (1, 0), (0, 1)]]])
    sa, sp, _ = run(ctx, arr, True)
    ua, _, _ = run(ctx, arr, False)
    assert abs(sa[0] - 24952305678.0) < 1 and abs(sp[0] - 631819.8745) < 1e-4 and sa[1] == -sa[0]
    assert rel(ua[0] + ua[1], R.AREA0) < 1e-15
    assert abs(sa[2] - 24619419146.0) < 1 and abs(sp[2] - 627598.2731) < 1e-4


def star(rng, cx, cy, r, k):
    t = np.sort(rng.uniform(0, 2 * np.pi, k))
    rr = r * rng.uniform(0.5, 1.0, k)
    c = max(np.cos(np.radians(cy)), 0.2)
    return [(cx + rr[i] * np.cos(t[i]) / c, cy + rr[i] * np.sin(t[i])) for i in range(k)]


def random_polygon(rng):
    cx, cy = rng.uniform(-180, 540), rng.uniform(-75, 75)
    r = min(10.0 ** rng.uniform(-5, 1.4), 89.0 - abs(cy))  # about 1 m to continental, |lat| < 89
    ext = star(rng, cx, cy, r, int(rng.integers(3, 40)))
    if rng.random() < 0.5:
        ext = ext[::-1]
    rings = [ext]
    for _ in range(int(rng.integers(0, 3))):
        h = star(rng, cx + rng.uniform(-0.1, 0.1) * r, cy + rng.uniform(-0.1, 0.1) * r, 0.2 * r, int(rng.integers(3, 12)))
        rings.append(h if rng.random() < 0.5 else h[::-1])
    if rng.random() < 0.3:
        rings = [ring + [ring[0]] for ring in rings]
    return rings


@pytest.mark.parametrize("signed", [True, False])
def test_random_polygons_and_multipolygons(ctx, signed):
    rng = np.random.default_rng(21 + signed)
    polys = [random_polygon(rng) for _ in range(300)]
    assert_matches(run(ctx, GeoArrowArray.from_shapes(P, polys), signed), R.geodesic_area(polys, "polygon", signed))
    multis = [[random_polygon(rng) for _ in range(int(rng.integers(0, 4)))] for _ in range(150)]
    assert_matches(run(ctx, GeoArrowArray.from_shapes(MP, multis), signed), R.geodesic_area(multis, "multipolygon", signed))


def test_nulls_empties_and_out_of_range_rows(ctx):
    sq = [(0, 0), (1, 0), (1, 1), (0, 1)]
    rows = [[sq], None, [], [[(0, 0), (1, np.nan), (1, 1)]], [[(0, 0), (np.inf, 0), (1, 1)]], [[(0, 0), (1, 90.5), (1, 1)]],
            [sq, [(0.2, 0.2), (0.2, -91), (0.4, 0.4)]], [[(10, 10)]], [sq]]
    a, p, v = run(ctx, GeoArrowArray.from_shapes(P, rows))
    assert v.tolist() == [True, False, True, False, False, False, False, True, True]
    assert a[2] == 0 and p[2] == 0 and a[7] == 0 and p[7] == 0 and a[0] == a[8] and a[0] > 0
    assert_matches((a, p, v), R.geodesic_area(rows, "polygon"))
    m = [[[sq]], [], None, [[sq], [[(0, 0), (1, -95), (1, 1)]]]]
    a, p, v = run(ctx, GeoArrowArray.from_shapes(MP, m))
    assert v.tolist() == [True, True, False, False] and a[1] == 0
    for t, shapes in [
        (GeometryType.POINT, [(1.0, 2.0), (-170.0, -89.0), (3.0, 95.0), (np.nan, 1.0)]),
        (GeometryType.LINESTRING, [[(0, 0), (1, 1)], [], None, [(0, 0), (1, 100)]]),
        (GeometryType.MULTIPOINT, [[(0, 0), (1, 1)], [], None, [(0, np.nan)]]),
        (GeometryType.MULTILINESTRING, [[[(0, 0), (1, 1)]], [], None, [[(0, 0)], [(2, -90.01)]]]),
    ]:
        a, p, v = run(ctx, GeoArrowArray.from_shapes(t, shapes))
        assert v.tolist() == [True, True, False, False]
        assert a[:2].tolist() == [0.0, 0.0] and p[:2].tolist() == [0.0, 0.0]


def test_datasets(ctx):
    d = datasets.read_dataset("naturalearth_lowres").geometry.device
    host = d.to_host()
    for signed in (True, False):
        got = engine.geodesic_area(d, signed)
        assert_matches(got, R.geodesic_area(R.column_shapes(host), "multipolygon" if host.type == MP else "polygon", signed))
    # the bundled Natural Earth rings are clockwise (the shapefile convention): signed areas are negative, and the unsigned
    # form of each part is the ellipsoid's area minus the part, as in geo; -signed is the countries' area
    s, _, sv = engine.geodesic_area(d, True)
    assert sv.all() and (s < 0).all() and 1.2e14 < -s.sum() < 1.6e14
    # unsigned: each clockwise exterior gives A0 minus the country and each (counter-clockwise) hole A0 minus the hole, so
    # South Africa, whose hole is Lesotho, comes out negative: geo's arithmetic on wrongly wound rings, kept
    a, p, v = engine.geodesic_area(d, False)
    assert v.all() and (a < 0).sum() == 1
    # the accessor
    acc = datasets.read_dataset("naturalearth_lowres").geometry.geo.geodesic_area_unsigned()
    assert np.array_equal(acc.to_numpy(zero_copy_only=False), a)
    per = datasets.read_dataset("naturalearth_lowres").geometry.geo.geodesic_perimeter()
    assert np.array_equal(per.to_numpy(zero_copy_only=False), p)
    signed = datasets.read_dataset("naturalearth_lowres").geometry.geo.geodesic_area_signed()
    assert np.array_equal(signed.to_numpy(zero_copy_only=False), engine.geodesic_area(d, True)[0])
    # a projected column (metres) is not (lon, lat): every row null
    nybb = datasets.read_dataset("nybb").geometry
    assert nybb.geo.geodesic_area_signed().null_count == len(nybb.device)


def test_determinism_and_independence_of_the_batch(ctx):
    rng = np.random.default_rng(4)
    few = [random_polygon(rng) for _ in range(20)]
    many = [random_polygon(rng) for _ in range(100_000)]
    pos = rng.choice(100_000, 20, replace=False)
    for i, k in enumerate(pos):
        many[k] = few[i]
    big = ctx.upload(GeoArrowArray.from_shapes(P, many))
    a1, p1, v1 = engine.geodesic_area(big, True)
    a2, p2, v2 = engine.geodesic_area(big, True)
    assert a1.tobytes() == a2.tobytes() and p1.tobytes() == p2.tobytes() and np.array_equal(v1, v2)
    a, p, v = run(ctx, GeoArrowArray.from_shapes(P, few))
    assert a.tobytes() == a1[pos].tobytes() and p.tobytes() == p1[pos].tobytes()
    for i in range(3):
        one = run(ctx, GeoArrowArray.from_shapes(P, [few[i]]))
        assert one[0].tobytes() == a[i : i + 1].tobytes()


def test_perimeter_equals_geodesic_length_for_closed_single_rings(ctx):
    rng = np.random.default_rng(8)
    rows = []
    for _ in range(500):
        ring = random_polygon(rng)[0]
        rows.append([ring + [ring[0]]])
    d = ctx.upload(GeoArrowArray.from_shapes(P, rows))
    _, p, v = engine.geodesic_area(d, True)
    length, lv = engine.geodesic_length(d, "geodesic")
    assert v.all() and lv.all()
    assert np.all(np.abs(p - length) <= 1e-13 * length)


def test_more_edges_than_one_pass(ctx):
    """a column above 2^26 edges runs in row chunks; each row's value is the one it has in a small call"""
    n, k = 1_100_000, 64
    rng = np.random.default_rng(17)
    t = np.linspace(0, 2 * np.pi, k, endpoint=False)
    cx, cy = rng.uniform(-180, 180, n), rng.uniform(-60, 60, n)
    r = 0.01 * rng.uniform(0.5, 1.5, (n, 1))
    xy = np.stack([cx[:, None] + r * np.cos(t), cy[:, None] + r * np.sin(t)], -1).reshape(-1, 2)
    off = np.arange(0, n * k + 1, k, dtype=np.int64)
    big = GeoArrowArray.polygons(xy, off, np.arange(n + 1, dtype=np.int64))
    a, p, v = run(ctx, big)
    assert v.all() and (a > 0).all()
    chunk = (1 << 26) // k
    for lo in (0, chunk - 3, n - 5):
        rows = np.arange(lo, lo + 5)
        sub = GeoArrowArray.polygons(xy[lo * k : (lo + 5) * k], off[:6], np.arange(6, dtype=np.int64))
        sa, sp, _ = run(ctx, sub)
        assert sa.tobytes() == a[rows].tobytes() and sp.tobytes() == p[rows].tobytes()


def test_invalid_arguments(ctx):
    import ctypes as C

    d = ctx.upload(GeoArrowArray.from_shapes(P, [[[(0, 0), (1, 0), (1, 1)]]]))
    out = np.empty(1)
    lib = ctx.lib
    assert lib.gpl_geodesic_area(ctx._h, d._h, 0, None, None, None, 0) == -7
    assert lib.gpl_geodesic_area(ctx._h, d._h, 2, out.ctypes.data_as(C.c_void_p), None, None, 0) == -7
    assert lib.gpl_geodesic_area(ctx._h, d._h, 1, out.ctypes.data_as(C.c_void_p), None, None, 5) == -7
    assert lib.gpl_geodesic_area(ctx._h, None, 1, out.ctypes.data_as(C.c_void_p), None, None, 0) == -7


def radii(phi):
    s = math.sin(math.radians(phi))
    w = math.sqrt(1 - R.E2 * s * s)
    return R.A * (1 - R.E2) / w**3, R.A / w  # meridional M, prime-vertical N


def test_closed_form_identities(ctx):
    """the CPU reference's identities, on the GPU: chord-split additivity, holes as separate polygons, small squares against
    M N cos(phi), longitude conventions and the +-180 straddle"""
    rng = np.random.default_rng(3)
    rows, checks = [], []

    def add(*polygons):
        first = len(rows)
        rows.extend(polygons)
        return range(first, len(rows))

    for cy in (-60.0, 0.0, 45.0):
        pts = star(rng, 20.0, cy, 2.0, 24)
        c = (20.0, cy)
        w, p1, p2 = add([pts], [[c] + pts[0:13]], [[c] + pts[12:] + [pts[0]]])
        checks.append(("split", w, p1, p2))
    ext = [(0, 0), (4, 0), (4, 4), (0, 4)]
    h1 = [(1, 1), (1, 2), (2, 2), (2, 1)]
    h2 = [(3, 3), (3.5, 3), (3.5, 3.5), (3, 3.5)]
    rows.append([ext, h1, h2])
    holed = len(rows) - 1
    e, a1, a2 = add([ext], [h1], [h2])
    squares = {}
    for lat in (0, 30, 60, 85):
        d = 0.001
        (squares[lat],) = add([[(10.0, lat - d / 2), (10.0 + d, lat - d / 2), (10.0 + d, lat + d / 2), (10.0, lat + d / 2)]])
    east, west, at0 = star(rng, 30.0, 10.0, 3.0, 17), star(rng, -100.0, -20.0, 3.0, 17), star(rng, 0.0, 40.0, 2.0, 15)
    shifts = add([east], [[(x + 360.0, y) for x, y in east]], [[(x - 360.0, y) for x, y in east]], [west],
                 [[(x + 360.0, y) for x, y in west]], [at0], [[((x + 180.0) if x < 0 else (x - 180.0), y) for x, y in at0]])
    a, _, v = run(ctx, GeoArrowArray.from_shapes(P, rows))
    assert v.all()
    for _, w, p1, p2 in checks:
        assert rel(a[p1] + a[p2], a[w]) < 1e-9
    assert rel(a[holed], a[e] - abs(a[a1]) - abs(a[a2])) < 1e-12
    for lat, i in squares.items():
        M, Nn = radii(lat)
        assert rel(a[i], 0.001**2 * (math.pi / 180) ** 2 * M * Nn * math.cos(math.radians(lat))) < 1e-5
    s = list(shifts)
    for i in (s[1], s[2]):
        assert rel(a[i], a[s[0]]) < 1e-12
    assert rel(a[s[4]], a[s[3]]) < 1e-12 and rel(a[s[6]], a[s[5]]) < 1e-12


@pytest.mark.parametrize("k", [3, 31, 32, 33, 64, 100, 1000])
def test_closed_and_unclosed_rings_agree_bit_for_bit(ctx, k):
    """the repeated closing vertex adds a zero edge to one lane's sum; the result does not change in any bit, also for rings
    of 32 and more edges where that lane already holds a sum"""
    rng = np.random.default_rng(k)
    polys = []
    for _ in range(40):
        cx, cy = rng.uniform(-180, 180), rng.uniform(-70, 70)
        ext = star(rng, cx, cy, 10.0 ** rng.uniform(-4, 1), k)
        hole = star(rng, cx, cy, 0.0, 3)  # degenerate, at the centre: still a ring of the polygon
        polys.append([ext, hole] if rng.random() < 0.3 else [ext])
    closed = [[ring + [ring[0]] for ring in p] for p in polys]
    for signed in (True, False):
        ao, po, vo = run(ctx, GeoArrowArray.from_shapes(P, polys), signed)
        ac, pc, vc = run(ctx, GeoArrowArray.from_shapes(P, closed), signed)
        assert vo.all() and vc.all()
        assert ao.tobytes() == ac.tobytes() and po.tobytes() == pc.tobytes()
        mo = run(ctx, GeoArrowArray.from_shapes(MP, [polys[:3], polys[3:4]]), signed)
        mc = run(ctx, GeoArrowArray.from_shapes(MP, [closed[:3], closed[3:4]]), signed)
        assert mo[0].tobytes() == mc[0].tobytes() and mo[1].tobytes() == mc[1].tobytes()
