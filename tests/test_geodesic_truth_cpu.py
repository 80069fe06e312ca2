"""The 40-digit geodesic reference (tests/geodesic_truth.py) against published values, closed forms and an independent ODE
integration; the committed fixture (tests/golden/geodesic_truth.npz) against a recomputation by that reference; and the CPU
oracle's Karney and Vincenty solves, its haversine and the area reference tests/geodesic_area_reference.py against the
fixture, each within a bound set from its measured maximum error (tests/geodesic_truth_bounds.py records both).  No GPU
needed."""
import math

import mpmath as mp
import numpy as np
import pytest

import geodesic_area_reference as R
import geodesic_truth as T
from geodesic_truth_bounds import (
    AREA_K,
    EPS,
    KARNEY_BOUND_M,
    VINCENTY_BOUND_M,
    VINCENTY_NULLS_PER_FAMILY,
    area_bound,
    err,
    haversine_bound,
    load,
    polygon_rows,
)

QUARTER_MERIDIAN = 10001965.729  # WGS84, metres


@pytest.fixture(autouse=True)
def forty_digits():
    """the tests' own arithmetic on the reference's mpf values runs at its precision"""
    with mp.workdps(T.DPS):
        yield


# ---- the reference against published values and closed forms ----


def test_published_values():
    qm = T.inverse(0.0, 0.0, 0.0, 90.0)[0]
    assert abs(qm - QUARTER_MERIDIAN) < 1e-3
    assert abs(qm - T.B * mp.ellipe(-T.EP2)) < mp.mpf(10) ** -30 * qm
    assert abs(T.AREA0 - 4 * mp.pi * T.authalic_F(mp.mpf(1))) < mp.mpf(10) ** -30 * T.AREA0
    assert abs(float(T.AREA0) - R.AREA0) < 1e-15 * R.AREA0
    # Karney 2013: the direct example (lat1 = 40, alp1 = 30, s12 = 10 000 km; the end point published to 1e-11 degrees)
    s, a1, _, lam = T.inverse(0.0, 40.0, 137.84490004377, 41.79331020506)
    assert abs(s - 1e7) < 1e-6 and abs(a1 - 30) < 1e-9 and abs(lam - 137.84490004377) < 1e-20
    # Karney 2013 section 7: a near-antipodal pair
    assert abs(T.inverse(0.0, -30.0, 179.8, 29.9)[0] - mp.mpf("19989832.82761")) < 1e-5
    # geographiclib's planimeter: the ring at 89 degrees
    area, per, _ = T.ring([(0, 89), (90, 89), (180, 89), (270, 89)])
    assert abs(area - 24952305678) < 1 and abs(per - mp.mpf("631819.8745")) < 1e-4


def test_closed_forms():
    for dlam in (1e-9, 1.0, 90.0, 179.0, 179.39):
        s, a1, a2, _ = T.inverse(10.0, 0.0, 10.0 + dlam, 0.0)
        assert abs(s - T.A * mp.radians(mp.mpf(10.0 + dlam) - 10)) < mp.mpf(10) ** -28 * T.A and abs(a1 - 90) < 1e-12 and abs(a2 - 90) < 1e-12
    # past (1 - f) 180 degrees the shortest line leaves the equator and is shorter than the equator
    for dlam in (179.5, 179.9):
        s, a1, _, _ = T.inverse(0.0, 0.0, dlam, 0.0)
        assert s < T.A * mp.radians(dlam) and 90 < a1 < 180
    for lat1, lat2 in ((-10.0, 50.0), (0.0, 89.0), (-89.5, -3.25)):
        b1, b2 = (mp.atan((1 - T.F_) * mp.tan(mp.radians(x))) for x in (lat1, lat2))
        want = T.B * (mp.ellipe(b2, -T.EP2) - mp.ellipe(b1, -T.EP2))
        assert abs(T.inverse(7.0, lat1, 7.0, lat2)[0] - want) < mp.mpf(10) ** -28 * want
        over = T.B * (2 * mp.ellipe(mp.pi / 2, -T.EP2) + mp.ellipe(b1, -T.EP2) + mp.ellipe(b2, -T.EP2))
        over_n = T.B * (2 * mp.ellipe(mp.pi / 2, -T.EP2) - mp.ellipe(b1, -T.EP2) - mp.ellipe(b2, -T.EP2))
        assert abs(T.inverse(7.0, lat1, 187.0, lat2)[0] - min(over, over_n)) < mp.mpf(10) ** -28 * over
    qm = T.B * mp.ellipe(-T.EP2)
    for dlam in (1, 45, 90, 135):
        area, per, _ = T.ring([(0.0, 0.0), (dlam, 0.0), (0.0, 90.0)])
        assert abs(area - T.AREA0 * dlam / 720) < mp.mpf(10) ** -25 * T.AREA0
        assert abs(per - (T.A * mp.radians(dlam) + 2 * qm)) < mp.mpf(10) ** -25 * per
        area, _, _ = T.ring([(0.0, 0.0), (0.0, -90.0), (dlam, 0.0)])
        assert abs(area - T.AREA0 * dlam / 720) < mp.mpf(10) ** -25 * T.AREA0
        area, _, _ = T.ring([(0.0, 90.0), (dlam, 0.0), (0.0, 0.0)], signed=False)
        assert abs(area - T.AREA0 * (1 - mp.mpf(dlam) / 720)) < mp.mpf(10) ** -25 * T.AREA0


def test_ode_cross_check():
    """integrate the geodesic's ODE in (phi, lambda, alpha) over s12 from point 1 with the true alp1: it lands on point 2"""
    from scipy.integrate import solve_ivp

    a, e2 = float(T.A), float(T.E2)
    fx = load()
    pin, fam, s12 = fx["pair_in"], fx["pair_family"], fx["pair_s12"][:, 0]
    pick = np.flatnonzero((fam == 0) & (s12 > 1e4) & (s12 < 1.5e7) & (np.abs(pin[:, 1]) < 70) & (np.abs(pin[:, 3]) < 70))[:10]
    assert len(pick) == 10

    def rhs(_, y):
        phi, _, alp = y
        w = math.sqrt(1 - e2 * math.sin(phi) ** 2)
        m, n = a * (1 - e2) / w**3, a / w
        return [math.cos(alp) / m, math.sin(alp) / (n * math.cos(phi)), math.sin(alp) * math.tan(phi) / n]

    for i in pick:
        lon1, lat1, lon2, lat2 = pin[i]
        alp1 = float(fx["pair_alp1"][i, 0])
        sol = solve_ivp(rhs, (0, s12[i]), [math.radians(lat1), 0.0, math.radians(alp1)], method="DOP853", rtol=1e-13, atol=1e-15)
        phi, lam, _ = sol.y[:, -1]
        w = math.sqrt(1 - e2 * math.sin(phi) ** 2)
        dlam = math.remainder(lam - math.radians(lon2 - lon1), 2 * math.pi)
        miss = math.hypot((phi - math.radians(lat2)) * a * (1 - e2) / w**3, dlam * a / w * math.cos(phi))
        assert miss < 1e-6, (i, miss)


# ---- the fixture is what the committed reference produces ----


def _close(got, want, scale):
    return abs(got - (mp.mpf(want[0]) + mp.mpf(want[1]))) <= mp.mpf(10) ** -25 * scale


def test_fixture_pairs_recompute():
    fx = load()
    rng = np.random.default_rng(5)
    for f in range(int(fx["pair_family"].max()) + 1):
        idx = np.flatnonzero(fx["pair_family"] == f)
        for i in rng.choice(idx, min(20, len(idx)), replace=False):
            s, a1, a2, lam, e = T.inverse(*fx["pair_in"][i], with_area=True)
            hav, _ = T.haversine(*fx["pair_in"][i])
            assert _close(s, fx["pair_s12"][i], max(s, 1e-300)), i
            assert _close(a1, fx["pair_alp1"][i], 180) and _close(a2, fx["pair_alp2"][i], 180), i
            assert _close(lam, fx["pair_lam12"][i], 180), i
            assert _close(e, fx["pair_E12"][i], T.AREA0), i
            assert _close(hav, fx["pair_haversine"][i], max(hav, 1e-300)), i


def test_fixture_polygons_recompute():
    """a seeded sample of edges of every polygon family recomputed, and every row's area and perimeter re-summed from the
    stored edges by the committed ring and polygon rules"""
    fx = load()
    xy, ro, po, wo, eo, edge = fx["poly_xy"], fx["poly_ring_off"], fx["poly_part_off"], fx["poly_row_off"], fx["poly_edge_off"], fx["poly_edge"]
    rng = np.random.default_rng(6)
    # ring -> row
    rows_of_ring = np.empty(len(ro) - 1, dtype=np.int64)
    for w in range(len(wo) - 1):
        rows_of_ring[po[wo[w]]:po[wo[w + 1]]] = w
    for f in range(int(fx["poly_family"].max()) + 1):
        rings = np.flatnonzero(fx["poly_family"][rows_of_ring] == f)
        for r in rng.choice(rings, min(20, len(rings)), replace=False):
            pts = [tuple(p) for p in xy[ro[r]:ro[r + 1]]]
            if len(pts) >= 2 and pts[-1] == pts[0]:
                pts = pts[:-1]
            j = int(rng.integers(len(pts)))
            p, q = pts[j], pts[(j + 1) % len(pts)]
            s, _, _, lam, e = T.inverse(p[0], p[1], q[0], q[1], with_area=True)
            want = edge[eo[r] + j]
            assert _close(s, want[0], max(s, 1e-300)) and _close(e, want[1], T.AREA0) and _close(lam, want[2], 180), (r, j)
    for w in range(len(wo) - 1):
        sig = uns = per = mp.mpf(0)
        for p in range(wo[w], wo[w + 1]):
            rs, ru = [], []
            for r in range(po[p], po[p + 1]):
                e = [tuple(mp.mpf(v[0]) + mp.mpf(v[1]) for v in ed) for ed in edge[eo[r]:eo[r + 1]]]
                rs.append(T.ring_from_edges(e, r > po[p], True))
                ru.append(T.ring_from_edges(e, r > po[p], False))
            a_s, pp = T.polygon_from_rings(rs)
            sig, uns, per = sig + a_s, uns + T.polygon_from_rings(ru)[0], per + pp
        scale = T.AREA0  # the stored edges carry ~1e-32 relative of terms up to area0, summed over a few dozen edges
        assert _close(sig, fx["poly_area_signed"][w], scale) and _close(uns, fx["poly_area_unsigned"][w], scale), w
        assert _close(per, fx["poly_perimeter"][w], per), w


# ---- the oracle against the fixture ----


def test_oracle_karney_and_vincenty(og):
    fx = load()
    pin, s12 = fx["pair_in"], fx["pair_s12"]
    k = np.array([og.geodesic_distance("geodesic", *p) for p in pin])
    v = np.array([og.geodesic_distance("vincenty", *p) for p in pin])
    assert np.abs(err(k, s12)).max() <= KARNEY_BOUND_M
    ok = ~np.isnan(v)
    assert np.abs(err(v[ok], s12[ok])).max() <= VINCENTY_BOUND_M
    # Vincenty fails to converge on near-antipodal pairs (and on the equator past (1 - f) 180 degrees) only
    fails = np.bincount(fx["pair_family"][~ok], minlength=len(np.unique(fx["pair_family"])))
    assert fails.tolist() == VINCENTY_NULLS_PER_FAMILY


def test_oracle_haversine(og):
    fx = load()
    pin = fx["pair_in"]
    h = np.array([og.geodesic_distance("haversine", *p) for p in pin])
    bound = haversine_bound(*pin.T)
    ok = ~np.isnan(h)
    assert np.all(np.abs(err(h[ok], fx["pair_haversine"][ok])) <= bound[ok])


def test_area_reference_pairs_and_polygons():
    """geodesic_area_reference's per-edge S12 and ring sums against the truth"""
    fx = load()
    pin, fam = fx["pair_in"], fx["pair_family"]
    for i in range(len(pin)):
        s, S12, mag = R.inverse(*pin[i])
        assert abs(err(s, fx["pair_s12"][i])) <= KARNEY_BOUND_M, i
        if fam[i] in (0, 1, 4) and fx["pair_s12"][i, 0] < 1.95e7:
            # over a pole geographiclib's S12 and the edge integral differ by area0 / 2 (which pole is a convention)
            d = abs(math.remainder(err(S12, fx["pair_E12"][i]), R.AREA0 / 2))
            assert d <= AREA_K * EPS * mag, i
    rows = polygon_rows(fx)
    multi = fx["poly_multi"]
    for signed, key in ((True, "poly_area_signed"), (False, "poly_area_unsigned")):
        for m, kind in ((False, "polygon"), (True, "multipolygon")):
            sel = np.flatnonzero(multi == m)
            a, p, v, scale = R.geodesic_area([rows[i] for i in sel], kind, signed)
            assert v.all()
            assert np.all(np.abs(err(a, fx[key][sel])) <= area_bound(fx, sel, scale, signed))
            edges = np.diff(fx["poly_edge_off"][fx["poly_part_off"][fx["poly_row_off"]]])[sel]
            assert np.all(np.abs(err(p, fx["poly_perimeter"][sel])) <= KARNEY_BOUND_M * edges)


