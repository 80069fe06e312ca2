"""The fixture of true geodesic values (tests/golden/geodesic_truth.npz, written by tests/golden/make_geodesic_truth.py from
tests/geodesic_truth.py) and the error bounds the CPU oracle and the GPU kernels are held to against it — numpy only, shared
by tests/test_geodesic_truth_cpu.py and tests/test_gpu_geodesic_truth.py.

Each bound is set from the maximum error measured on the CPU oracle over the whole fixture (x86-64, libm), recorded beside
it; the maxima measured on the GPU are in the GPU test."""
import os

import numpy as np

import geodesic_area_reference as R

FIXTURE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "geodesic_truth.npz")
EPS = 2.0**-52
PAIR_FAMILIES = ["random", "tiny", "equator", "meridian", "pole", "antipodal", "shifted", "swapped"]
POLY_FAMILIES = ["star", "multi", "antimeridian", "special", "pole", "large"]

# Karney's inverse (the oracle's distance solve and geodesic_area_reference's): max |ds| = 6.3e-9 m over 2 818 pairs
KARNEY_BOUND_M = 1e-8
# Vincenty, where it converges: max |ds| = 7.9e-5 m (a near-antipodal pair); it is null on 645 pairs, all near-antipodal or
# equatorial past (1 - f) 180 degrees
VINCENTY_BOUND_M = 2e-4
VINCENTY_NULLS_PER_FAMILY = [0, 0, 108, 0, 0, 348, 99, 90]  # in PAIR_FAMILIES order
# haversine: |dd| <= K eps R (1 + (|lon1| + |lon2|) / 180 + 1 / sqrt(1 - a)), measured K = 2.0 (1.7 on the 1 018 pairs
# under 100 m; a law-of-cosines distance needs K = 3e7)
HAVERSINE_K = 4.0
# polygon area: |dA| <= AREA_K eps (scale + |A|) signed, AREA_K eps (scale + rings area0) unsigned, where scale sums the
# magnitudes of the terms of every S12 (geodesic_area_reference) and an unsigned ring's reduction to [0, area0) can leave a
# rounding of area0 in the result; geodesic_area_reference measures 10.5 (signed, the near-antipodal edges) and 1.0
# (unsigned).  Per edge, for the random, tiny and polar pairs short of the antipode (s12 < 19 500 km): |dS12| <= AREA_K eps
# scale, measured 5.7.  Near the antipode and on nearly meridional lines S12 is ill-conditioned: the azimuths, and with
# them the area term, swing with the last bits of the input (up to 1.3e3 eps scale), so those are checked per ring only.
AREA_K = 16.0


def load():
    return np.load(FIXTURE)


def err(got, truth):
    """got - truth for doubles got and (hi, lo) truths"""
    return (np.asarray(got, dtype=np.float64) - truth[..., 0]) - truth[..., 1]


def haversine_bound(lon1, lat1, lon2, lat2):
    """K eps R (1 + (|lon1| + |lon2|) / 180 + 1 / sqrt(1 - a)) for geo's 2 R asin(sqrt(a)).  Every input of a is a difference
    of coordinates or a latitude, rounded relative to itself, so a carries a relative error of a few eps and the distance an
    absolute one of about eps R (1 + 1 / sqrt(1 - a)): the last term is asin's conditioning at the antipode.  A longitude
    difference of more than a turn (inputs such as 690 and -30) is rounded relative to its size before sin takes it modulo
    2 pi, which the |lon| / 180 terms cover.  A short pair is held to a few eps R absolute, far below its length, so an
    expression that cancels there (the law of cosines, off by centimetres) fails."""
    p1, p2 = np.radians(lat1), np.radians(lat2)
    a = np.sin((p2 - p1) / 2) ** 2 + np.cos(p1) * np.cos(p2) * np.sin(np.radians(lon2 - lon1) / 2) ** 2
    return HAVERSINE_K * EPS * 6371008.8 * (1 + (np.abs(lon1) + np.abs(lon2)) / 180 + 1 / np.sqrt(np.maximum(1 - a, EPS * EPS)))


def area_bound(fx, sel, scale, signed):
    rings = np.diff(fx["poly_part_off"][fx["poly_row_off"]])[sel]
    return AREA_K * EPS * (scale + (np.abs(fx["poly_area_signed"][sel, 0]) if signed else rings * R.AREA0))


def polygon_rows(fx):
    """the fixture's polygon rows as nested lists (Polygon rows: [ring]; MultiPolygon rows: [[ring]])"""
    xy, ro, po, wo = fx["poly_xy"], fx["poly_ring_off"], fx["poly_part_off"], fx["poly_row_off"]
    rows = []
    for i in range(len(wo) - 1):
        polys = [[xy[ro[r]:ro[r + 1]].tolist() for r in range(po[p], po[p + 1])] for p in range(wo[i], wo[i + 1])]
        rows.append(polys if fx["poly_multi"][i] else polys[0])
    return rows
