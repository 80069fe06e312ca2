"""CPU model of the window of the great-circle joins (geo_window / geo_split in k_geo_join.cu, DESIGN.md §4.15), restated in
Python doubles.

A left point (lon, lat) walks the grid rows [cell(lat - dlat), cell(lat + dlat)] and, unless the band reaches a pole, the
columns of the longitudes within dlon = asin(sin delta / cos lat) of its wrapped longitude, delta = (D / R)(1 + REL) + ABS.
An interval that passes +-180 becomes two column ranges; a part that lies outside the union box is dropped and two parts
that meet in cell space become the whole row of cells, so that no cell is listed twice.  Checked here on adversarial inputs:
  * every eligible right row whose computed haversine distance is <= D lies in a cell of the window;
  * no cell is visited twice.
Negative controls, each found by a seeded search: without the slack (REL = ABS = 0) a row at distance exactly D falls outside
the window, and with the two parts of a split taken as clamped cell ranges without the disjointness rule a cell is visited
twice."""
import math

import numpy as np

from test_nearest_bound_model import jg_cell

R = 6371008.8
DEG = 0.017453292519943295769
REL, ABS, WHOLE, POLE, LONPAD = 2.0 ** -36, 1e-12, 1.0, 1e-9, 1e-9
HALF_PI = 1.57079632679489661923
CIRC_HALF = math.pi * R


def haversine(p, q):
    """the expression of haversine.cuh with libm's sin / cos / asin; NaN where a > 1"""
    th1, th2 = p[1] * DEG, q[1] * DEG
    dth, dla = (q[1] - p[1]) * DEG, (q[0] - p[0]) * DEG
    s1, s2 = math.sin(dth / 2.0), math.sin(dla / 2.0)
    a = s1 * s1 + math.cos(th1) * math.cos(th2) * (s2 * s2)
    return R * (2.0 * math.asin(math.sqrt(a))) if a <= 1.0 else math.nan


def eligible(p):
    return abs(p[1]) <= 90.0 and abs(p[0]) <= 360.0


def wrap(lon):
    return lon - 360.0 if lon >= 180.0 else (lon + 360.0 if lon < -180.0 else lon)


class Grid:
    """the grid gpl_geo_index_build makes of the eligible rows; g defaults to ceil(sqrt(rows)) capped at 2048"""

    def __init__(self, rows, g=None):
        self.rows = [q for q in rows if eligible(q)]
        xs, ys = [wrap(q[0]) for q in self.rows], [q[1] for q in self.rows]
        self.ux0, self.ux1, self.uy0, self.uy1 = min(xs), max(xs), min(ys), max(ys)
        self.g = g or min(2048, max(1, math.ceil(math.sqrt(len(self.rows)))))
        w, h = self.ux1 - self.ux0, self.uy1 - self.uy0
        self.iw = self.g / w if w > 0 and math.isfinite(self.g / w) else 0.0
        self.ih = self.g / h if h > 0 and math.isfinite(self.g / h) else 0.0
        self.gx = 1 if self.iw == 0.0 else self.g
        self.gy = 1 if self.ih == 0.0 else self.g

    def cx(self, v):
        return jg_cell(v, self.ux0, self.iw, self.g)

    def cy(self, v):
        return jg_cell(v, self.uy0, self.ih, self.g)

    def cell_of(self, q):
        return self.cx(wrap(q[0])), self.cy(q[1])


def window(G, p, D, rel=REL, abs_=ABS, disjoint=True):
    """the visited cells as (cy0, cy1, [column runs]); None when empty"""
    delta = (D / R) * (1.0 + rel) + abs_
    if not delta <= WHOLE:
        return 0, G.gy - 1, [(0, G.gx - 1)]
    dlat = delta / DEG * (1.0 + rel)
    lat_lo, lat_hi = p[1] - dlat, p[1] + dlat
    if lat_lo > G.uy1 or lat_hi < G.uy0:
        return None
    cy0, cy1 = G.cy(lat_lo), G.cy(lat_hi)
    if abs(p[1]) * DEG + delta >= HALF_PI - POLE:
        return cy0, cy1, [(0, G.gx - 1)]
    ratio = math.sin(delta) / math.cos(p[1] * DEG) * (1.0 + rel)
    dlon = math.asin(min(ratio, 1.0)) / DEG * (1.0 + rel) + (LONPAD if abs_ else 0.0)
    wl = wrap(p[0])
    lo, hi = wl - dlon, wl + dlon
    if lo < -180.0:
        east_from, west_to = lo + 360.0, hi
    elif hi >= 180.0:
        east_from, west_to = lo, hi - 360.0
    else:
        if lo > G.ux1 or hi < G.ux0:
            return None
        return cy0, cy1, [(G.cx(lo), G.cx(hi))]
    ce, cw = G.cx(east_from), G.cx(west_to)
    if not disjoint:  # the two parts as clamped cell ranges, nothing else
        return cy0, cy1, [(ce, G.gx - 1), (0, cw)]
    east, west = east_from <= G.ux1, west_to >= G.ux0
    if east and west:
        runs = [(0, G.gx - 1)] if cw >= ce else [(ce, G.gx - 1), (0, cw)]  # the kernel's cx0 = ce, cx1 = gx + cw
    elif east:
        runs = [(ce, G.gx - 1)]
    elif west:
        runs = [(0, cw)]
    else:
        return None
    return cy0, cy1, runs


def columns(w):
    """the columns visited in each grid row of the window, in order (the rows cy0 .. cy1 are one range: only a column can
    come twice)"""
    return [] if w is None else [cx for a, b in w[2] for cx in range(a, b + 1)]


def lost_rows(G, p, D, **kw):
    """eligible rows with computed distance <= D whose cell the window does not visit"""
    w = window(G, p, D, **kw)
    if w is None:
        return [q for q in G.rows if haversine(p, q) <= D]
    cy0, cy1, runs = w
    out = []
    for q in G.rows:
        if haversine(p, q) <= D:
            cx, cy = G.cell_of(q)
            if not (cy0 <= cy <= cy1 and any(a <= cx <= b for a, b in runs)):
                out.append(q)
    return out


def ulps(v):
    return [math.nextafter(v, -math.inf), v, math.nextafter(v, math.inf)]


def special_points():
    lons = [v for b in (-180.0, 180.0, 0.0, 360.0, -360.0, 359.9, 180.1, -179.9, 90.0) for v in ulps(b) if abs(v) <= 360.0]
    lats = [v for b in (-90.0, 90.0, 0.0, 89.999999, -89.999999, 60.0, -45.0) for v in ulps(b) if abs(v) <= 90.0]
    return [(x, y) for x in lons for y in lats]


def distances_for(p, q):
    d = haversine(p, q)
    out = [1e-3, 1.0, 500.0, 1e4, 1e6, WHOLE * R * 0.999, WHOLE * R * 1.001, CIRC_HALF / 2, CIRC_HALF]
    if d == d:
        out += [v for v in ulps(d) if 0.0 <= v]
    return out


def check_sound(G, p, D):
    assert lost_rows(G, p, D) == [], (p, D)
    w = window(G, p, D)
    c = columns(w)
    assert len(c) == len(set(c)) and (w is None or w[0] <= w[1]), (p, D)


def test_window_holds_every_row_within_D_on_adversarial_inputs():
    pts = special_points()
    rng = np.random.default_rng(15)
    rows = pts + [(float(x), float(y)) for x, y in zip(rng.uniform(-180, 360, 300), np.degrees(np.arcsin(rng.uniform(-1, 1, 300))))]
    rows += [(math.nan, 0.0), (0.0, 91.0), (361.0, 0.0), (math.inf, 1.0)]  # never listed
    for g in (None, 7, 2048):
        G = Grid(rows, g)
        assert all(eligible(q) for q in G.rows) and len(G.rows) == len(rows) - 4
        for p in pts[::5] + [(179.99999, 0.0), (-179.99999, 0.0), (10.0, 89.9999999), (359.99999, -89.9999999)]:
            for q in (pts[3], pts[-7], rows[len(pts) + 3], (wrap(p[0] + 180.0), -p[1])):
                for D in distances_for(p, q):
                    check_sound(G, p, D)


def test_antimeridian_and_0_360_rows_are_found():
    east = [(179.95 + 0.001 * k, 0.02 * k - 0.1) for k in range(40)]  # some beyond 180: the 0..360 convention
    west = [(-179.95 - 0.001 * k, 0.02 * k - 0.1) for k in range(40)]
    for rows in (east + west, [(x + 360.0 if x < 0 else x, y) for x, y in east + west]):
        G = Grid(rows, 16)
        for p in ((179.9, 0.0), (-179.9, 0.0), (180.0, 0.0), (-180.0, 0.0), (180.1, 0.05), (math.nextafter(180.0, 0.0), 0.0)):
            for D in (0.0, 1e3, 22e3, 2.3e4, 1e5):
                check_sound(G, p, D)
            near = [wrap(q[0]) > 0 for q in G.rows if haversine(p, q) <= 3e4]
            assert any(near) and not all(near)  # rows on both sides of the line are within reach


def test_polar_caps_take_every_longitude():
    rows = [(float(x), 89.9) for x in range(-180, 180, 7)] + [(0.0, 90.0), (123.0, -90.0)] + [(float(x), -89.95) for x in range(0, 360, 11)]
    G = Grid(rows, 32)
    for p in ((0.0, 90.0), (77.0, math.nextafter(90.0, 0.0)), (-140.0, 89.95), (10.0, -90.0), (200.0, -89.99)):
        for D in (0.0, 1.0, 5e3, 1.2e4, 2e4, 1e5):
            check_sound(G, p, D)
        w = window(G, p, 2e4)
        assert w[2] == [(0, G.gx - 1)]


def test_union_box_much_smaller_than_the_globe():
    rng = np.random.default_rng(16)
    rows = [(float(x), float(y)) for x, y in zip(rng.uniform(10.0, 10.5, 400), rng.uniform(50.0, 50.2, 400))]
    G = Grid(rows)
    lefts = rows[:20] + [(9.9, 50.1), (10.6, 50.1), (10.2, 49.9), (10.2, 50.3), (-170.0, 50.1), (190.2, 50.1), (10.2, -50.0), (370.0, 50.0)]
    for p in lefts:
        if not eligible(p):
            continue
        for D in (0.0, 10.0, 500.0, 5e3, 5e4, 1e6, CIRC_HALF):
            check_sound(G, p, D)
    assert window(G, (-170.0, 50.1), 5e3) is None and window(G, (10.2, -50.0), 5e3) is None
    # degenerate grids: one row, one meridian, one parallel
    for rows in ([(179.5, 10.0)], [(180.0, float(y)) for y in range(-80, 81, 10)], [(float(x), 0.0) for x in range(-180, 180, 10)]):
        G = Grid(rows)
        for p in ((179.9, 10.0), (-179.9, 10.0), (-180.0, 0.0), (0.0, 0.0)):
            for D in (0.0, 5e4, 2e5, 5e6, CIRC_HALF):
                check_sound(G, p, D)


def test_negative_control_no_slack_loses_a_row():
    """a right row on an exact cell boundary at the easternmost longitude of a cap that nearly reaches the pole, D = the
    pair's computed distance: asin is steep there, and with REL = ABS = 0 the rounded eastern edge falls west of the row for
    some seeds; with the slack it never does"""
    frame = [(-128.0, -80.0), (128.0, 80.0)]  # 2048 columns of 1/8 degree: boundaries and cells are exact west of -64
    rng = np.random.default_rng(17)
    lost = 0
    for _ in range(300):
        phi = float(rng.uniform(50.0, 70.0))
        d0 = (90.0 - phi - float(rng.uniform(1e-5, 1e-3))) * DEG
        qx = -128.0 + int(rng.integers(8, 500)) / 8
        qy = math.degrees(math.asin(math.sin(phi * DEG) / math.cos(d0)))
        p = (qx - math.degrees(math.asin(math.sin(d0) / math.cos(phi * DEG))), phi)
        if p[0] < -180.0:
            continue
        G = Grid(frame + [(qx, qy)], 2048)
        D = haversine(p, (qx, qy))
        assert lost_rows(G, p, D) == []
        lost += len(lost_rows(G, p, D, rel=0.0, abs_=0.0))
    assert lost > 0


def test_negative_control_split_without_the_disjointness_rule_visits_a_cell_twice():
    """a union box just east of the antimeridian and left points just west of it: the eastern part of a split interval lies
    beyond the box and clamps to its last column, which the western part reaches too"""
    rng = np.random.default_rng(18)
    rows = [(float(x), float(y)) for x, y in zip(rng.uniform(-179.0, -170.0, 50), rng.uniform(-10.0, 10.0, 50))]
    G = Grid(rows)
    twice = 0
    for _ in range(200):
        p = (float(rng.uniform(175.0, 180.0)), float(rng.uniform(-10, 10)))
        D = float(rng.uniform(2e6, 6e6))
        c = columns(window(G, p, D))
        assert len(c) == len(set(c))
        assert lost_rows(G, p, D) == []
        bad = columns(window(G, p, D, disjoint=False))
        twice += len(bad) != len(set(bad))
    assert twice > 0
