"""The CPU reference for geodesic area and perimeter (tests/geodesic_area_reference.py) against closed forms and published
geographiclib values.  No GPU needed."""
import math

import numpy as np
import pytest

import geodesic_area_reference as R

QUARTER_MERIDIAN = 10001965.729  # WGS84, metres


def rel(a, b):
    return abs(a - b) / max(abs(a), abs(b), 1e-300)


def triangle(dlam):
    return [(0.0, 0.0), (dlam, 0.0), (0.0, 90.0)]


@pytest.mark.parametrize("dlam", [1, 45, 90, 135])
def test_pole_equator_triangles(dlam):
    want = R.AREA0 * dlam / 720
    area, per, _ = R.ring(triangle(dlam))
    assert rel(area, want) < 1e-13
    assert abs(per - (R.A * dlam * math.pi / 180 + 2 * QUARTER_MERIDIAN)) < 1e-3
    rev = list(reversed(triangle(dlam)))
    assert rel(R.ring(rev)[0], -want) < 1e-13
    assert rel(R.ring(rev, sign=False)[0], R.AREA0 - want) < 1e-13
    south = [(0.0, 0.0), (0.0, -90.0), (dlam, 0.0)]
    assert rel(R.ring(south)[0], want) < 1e-13


def test_published_values():
    """geographiclib's planimeter checks (points given there as (lat, lon))"""
    assert abs(R.AREA0 / 8 - 63758202715511.0) < 1
    a, p, _ = R.ring([(0, 89), (90, 89), (180, 89), (270, 89)])
    assert abs(a - 24952305678.0) < 1 and abs(p - 631819.8745) < 1e-4
    a, p, _ = R.ring([(0, -89), (90, -89), (180, -89), (270, -89)])
    assert abs(a + 24952305678.0) < 1 and abs(p - 631819.8745) < 1e-4
    a, p, _ = R.ring([(-1, 0), (0, -1), (1, 0), (0, 1)])
    assert abs(a - 24619419146.0) < 1 and abs(p - 627598.2731) < 1e-4
    a, p, _ = R.ring([(0, 90), (0, 0), (90, 0)])
    assert abs(a - 63758202715511.0) < 1 and abs(p - 30022685) < 1
    assert abs(R.inverse(0, -30, 179.8, 29.9)[0] - 19989832.82761) < 1e-4


def test_polar_ring_both_windings():
    ring = [(0, 89), (90, 89), (180, 89), (270, 89)]
    rev = list(reversed(ring))
    u1, u2 = R.ring(ring, sign=False)[0], R.ring(rev, sign=False)[0]
    assert rel(u1 + u2, R.AREA0) < 1e-15
    assert R.ring(ring)[0] == -R.ring(rev)[0]


def star(rng, cx, cy, r, k):
    t = np.sort(rng.uniform(0, 2 * np.pi, k))
    rr = r * rng.uniform(0.5, 1.0, k)
    return [(cx + rr[i] * np.cos(t[i]) / np.cos(np.radians(cy)), cy + rr[i] * np.sin(t[i])) for i in range(k)]


def test_additivity_of_a_chord_split():
    """a star-shaped ring split along a chord from its centre: the pieces' areas sum to the whole"""
    rng = np.random.default_rng(3)
    for cy in (-60.0, 0.0, 45.0):
        pts = star(rng, 20.0, cy, 2.0, 24)
        c = (20.0, cy)
        whole = R.ring(pts)[0]
        # split at vertices 0 and 12 through the centre: two polygons sharing the two chords c-p0 and c-p12
        p1 = [c] + pts[0:13]
        p2 = [c] + pts[12:] + [pts[0]]
        a1, a2 = R.ring(p1)[0], R.ring(p2)[0]
        assert rel(a1 + a2, whole) < 1e-9


def test_holes_subtract():
    ext = [(0, 0), (4, 0), (4, 4), (0, 4)]
    h1 = [(1, 1), (1, 2), (2, 2), (2, 1)]  # clockwise
    h2 = [(3, 3), (3.5, 3), (3.5, 3.5), (3, 3.5)]  # counter-clockwise: holes count by magnitude
    a, p, _ = R.polygon([ext, h1, h2])
    e = R.ring(ext)
    want = e[0] - abs(R.ring(h1)[0]) - abs(R.ring(h2)[0])
    assert rel(a, want) < 1e-15
    assert rel(p, e[1] + R.ring(h1)[1] + R.ring(h2)[1]) < 1e-15
    # a clockwise exterior: the hole sum is negated, so the signed result is sign(E) (|E| - H)
    a2, _, _ = R.polygon([list(reversed(ext)), h1, h2])
    assert rel(a2, -want) < 1e-12


def radii(phi):
    s = math.sin(math.radians(phi))
    w = math.sqrt(1 - R.E2 * s * s)
    return R.A * (1 - R.E2) / w**3, R.A / w  # M, N


@pytest.mark.parametrize("lat", [0, 30, 60, 85])
def test_small_squares(lat):
    d = 0.001
    sq = [(10.0, lat - d / 2), (10.0 + d, lat - d / 2), (10.0 + d, lat + d / 2), (10.0, lat + d / 2)]
    M, Nn = radii(lat)
    want = d * d * (math.pi / 180) ** 2 * M * Nn * math.cos(math.radians(lat))
    assert rel(R.ring(sq)[0], want) < 1e-5


def test_longitude_conventions():
    rng = np.random.default_rng(5)
    pts = star(rng, 30.0, 10.0, 3.0, 17)
    a = R.ring(pts)[0]
    for shift in (360.0, -360.0):
        assert rel(R.ring([(x + shift, y) for x, y in pts])[0], a) < 1e-12
    west = star(rng, -100.0, -20.0, 3.0, 17)
    aw = R.ring(west)[0]
    assert rel(R.ring([(x + 360.0, y) for x, y in west])[0], aw) < 1e-12
    # across +-180 versus the same shape across 0
    shape = star(rng, 0.0, 40.0, 2.0, 15)
    at0 = R.ring(shape)[0]
    wrapped = [((x + 180.0) if x < 0 else (x - 180.0), y) for x, y in shape]  # straddles +-180, written in -180..180
    assert rel(R.ring(wrapped)[0], at0) < 1e-12


def test_closed_and_unclosed_rings_agree_bit_for_bit():
    rng = np.random.default_rng(9)
    pts = star(rng, -70.0, -35.0, 1.0, 11)
    open_ = R.ring(pts)
    closed = R.ring(pts + [pts[0]])
    assert open_[0] == closed[0] and open_[1] == closed[1]


def test_rows_nulls_and_other_types():
    sq = [(0, 0), (1, 0), (1, 1), (0, 1)]
    a, p, v, _ = R.geodesic_area([[sq], [], None, [[(0, 0), (1, float("nan")), (1, 1)]], [[(0, 0), (1, 91), (1, 1)]]], "polygon")
    assert v.tolist() == [True, True, False, False, False]
    assert a[1] == 0 and p[1] == 0 and a[0] > 0
    a, p, v, _ = R.geodesic_area([[[sq]], [[sq], [sq]], []], "multipolygon")
    assert v.all() and rel(a[1], 2 * a[0]) < 1e-15 and a[2] == 0
    a, p, v, _ = R.geodesic_area([(1.0, 2.0), (3.0, 95.0), None], "point")
    assert v.tolist() == [True, False, False] and a[0] == 0 and p[0] == 0
