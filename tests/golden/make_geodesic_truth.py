"""Writes tests/golden/geodesic_truth.npz: the true geodesic distances, azimuths, edge integrals and haversine distances of
about 3 000 (lon, lat) pairs, and the true geodesic area and perimeter of about 400 Polygon / MultiPolygon rows, computed by
tests/geodesic_truth.py at 40 digits.

    python tests/golden/make_geodesic_truth.py

Fixed seeds; the work is spread over every core (a few minutes on 8) and the output does not depend on how many there are.
Every truth is stored as a (hi, lo) pair of doubles with hi + lo the 40-digit value to about 1e-32 relative.  The file is an
uncompressed zip with fixed timestamps, so a rerun reproduces it byte for byte.
"""
import io
import multiprocessing
import os
import sys
import zipfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import geodesic_truth as T  # noqa: E402
from geodesic_truth_bounds import PAIR_FAMILIES, POLY_FAMILIES  # noqa: E402

OUT = os.path.join(HERE, "geodesic_truth.npz")


def _direct_sphere(lon, lat, az, d):
    """a rough spherical direct step, only to place the second point (the truth is the inverse of the doubles it gives)"""
    p, l, a = np.radians(lat), np.radians(lon), np.radians(az)
    p2 = np.arcsin(np.clip(np.sin(p) * np.cos(d) + np.cos(p) * np.sin(d) * np.cos(a), -1, 1))
    l2 = l + np.arctan2(np.sin(a) * np.sin(d) * np.cos(p), np.cos(d) - np.sin(p) * np.sin(p2))
    return (np.degrees(l2) + 180) % 360 - 180, np.degrees(p2)


def _sphere_point(rng, n):
    return rng.uniform(-180, 180, n), np.degrees(np.arcsin(rng.uniform(-1, 1, n)))


def make_pairs():
    rng = np.random.default_rng(20261017)
    rows, fam = [], []

    def add(f, lo1, la1, lo2, la2):
        rows.append((float(lo1), float(la1), float(lo2), float(la2)))
        fam.append(PAIR_FAMILIES.index(f))

    # uniform on the sphere, log-uniform lengths from 1 mm to 20 000 km
    lo1, la1 = _sphere_point(rng, 1100)
    d = 10.0 ** rng.uniform(-3, np.log10(2e7), 1100) / 6371008.8
    lo2, la2 = _direct_sphere(lo1, la1, rng.uniform(0, 360, 1100), d)
    for i in range(1100):
        add("random", lo1[i], la1[i], lo2[i], la2[i])
    random_rows = list(rows)
    # separations from 1e-9 to 1e-3 degrees, anywhere, near +-180 and above 89.9 degrees
    for i in range(300):
        sep, th = 10.0 ** rng.uniform(-9, -3), rng.uniform(0, 2 * np.pi)
        if i % 3 == 0:
            lo, la = rng.uniform(-180, 180), np.degrees(np.arcsin(rng.uniform(-1, 1)))
        elif i % 3 == 1:
            lo, la = rng.choice([-180.0, 180.0]) - np.sign(rng.uniform(-1, 1)) * 10.0 ** rng.uniform(-9, -3), rng.uniform(-80, 80)
        else:
            lo, la = rng.uniform(-180, 180), rng.choice([-1, 1]) * (90 - 10.0 ** rng.uniform(-7, -1))
        la2 = float(np.clip(la + sep * np.sin(th), -90, 90))
        add("tiny", lo, la, lo + sep * np.cos(th), la2)
    # the equator, on both sides of the (1 - f) 180 degree limit
    lim = float(T.EQ_LIMIT)
    dlams = [1e-9, 1.0, 90.0, 179.0, 179.3965 - 1e-6, 179.3965 + 1e-6, lim, np.nextafter(lim, 0), np.nextafter(lim, 360),
             lim - 1e-6, lim + 1e-6, 179.5, 179.9, 180.0]
    for dl in dlams:
        for lo in (0.0, -179.5, 37.25, 179.0):
            add("equator", lo, 0.0, lo + dl, 0.0)
            add("equator", lo, 0.0, lo - dl, 0.0)
            add("equator", lo + dl, 0.0, lo, 0.0)
    # meridians: the same longitude, and 180 degrees apart (over a pole)
    for i in range(150):
        lo = float(rng.integers(-720, 720)) / 4
        add("meridian", lo, rng.uniform(-90, 90), lo + (180.0 if i % 2 else 0.0), rng.uniform(-90, 90))
    # endpoints exactly at a pole, several longitudes
    for i in range(100):
        pl = 90.0 if i % 2 else -90.0
        lo = [0.0, 45.0, -120.0, 180.0, -180.0, 33.3][i % 6]
        other = (rng.uniform(-180, 180), rng.uniform(-90, 90)) if i % 10 else (rng.uniform(-180, 180), float(rng.choice([-90, 90])))
        if i % 4 < 2:
            add("pole", lo, pl, *other)
        else:
            add("pole", *other, lo, pl)
    # near-antipodal: lat2 ~ -lat1, lambda12 within 1e-6 to 1.5 degrees of 180, and Karney 2013 section 7's pair
    add("antipodal", 0.0, -30.0, 179.8, 29.9)
    for i in range(399):
        la = rng.uniform(-80, 80)
        off = 10.0 ** rng.uniform(-6, np.log10(1.5))
        lo = rng.uniform(-180, 180)
        add("antipodal", lo, la, lo + rng.choice([-1, 1]) * (180 - off), -la + rng.uniform(-1, 1) * 10.0 ** rng.uniform(-6, 0))
    antipodal_rows = rows[-400:]
    # longitudes shifted by +-360, 540 and -720 (both or one endpoint), and lambda12 = 180 exactly and +-1 ulp
    src = random_rows[:150] + antipodal_rows[:90]
    for i, (a, b, c, e) in enumerate(src):
        s1, s2 = [(360.0, 360.0), (-360.0, 0.0), (540.0, -180.0), (-720.0, 360.0), (0.0, 540.0), (-720.0, -720.0)][i % 6]
        add("shifted", a + s1, b, c + s2, e)
    for i in range(60):
        lo, la = float(rng.integers(-720, 720)) / 4, rng.uniform(-89, 89)
        lo2 = lo + 180.0
        lo2 = [lo2, np.nextafter(lo2, np.inf), np.nextafter(lo2, -np.inf)][i % 3]
        add("shifted", lo, la, lo2, rng.uniform(-89, 89) if i % 2 else -la)
    # swapped endpoints
    for a, b, c, e in random_rows[:200] + antipodal_rows[:100]:
        add("swapped", c, e, a, b)
    return np.array(rows, dtype=np.float64), np.array(fam, dtype=np.int8)


def _star(rng, cx, cy, r, k):
    t = np.sort(rng.uniform(0, 2 * np.pi, k))
    rr = r * rng.uniform(0.5, 1.0, k)
    c = max(np.cos(np.radians(cy)), 0.2)
    return [(float(cx + rr[i] * np.cos(t[i]) / c), float(cy + rr[i] * np.sin(t[i]))) for i in range(k)]


def _star_polygon(rng, cx=None, cy=None, rmax=1.4):
    cx = rng.uniform(-180, 540) if cx is None else cx
    cy = rng.uniform(-75, 75) if cy is None else cy
    r = min(10.0 ** rng.uniform(-5, rmax), 89.0 - abs(cy))
    ext = _star(rng, cx, cy, r, int(rng.integers(3, 9)))
    if rng.random() < 0.5:
        ext = ext[::-1]
    rings = [ext]
    for _ in range(int(rng.integers(0, 3))):
        h = _star(rng, cx + rng.uniform(-0.1, 0.1) * r, cy + rng.uniform(-0.1, 0.1) * r, 0.2 * r, int(rng.integers(3, 6)))
        rings.append(h if rng.random() < 0.5 else h[::-1])
    if rng.random() < 0.3:
        rings = [ring + [ring[0]] for ring in rings]
    return rings


def make_polygons():
    rng = np.random.default_rng(17102026)
    rows = []  # (family, multi, [polygon = [ring]])

    def add(f, polys, multi=False):
        rows.append((POLY_FAMILIES.index(f), multi, polys))

    for _ in range(120):
        add("star", [_star_polygon(rng)])
    for _ in range(50):
        add("multi", [_star_polygon(rng) for _ in range(int(rng.integers(1, 4)))], True)
    for i in range(50):
        cx = [180.0, -180.0, 0.0, 360.0, 540.0][i % 5]
        p = _star_polygon(rng, cx, rng.uniform(-60, 60), 0.5)
        snap = [180.0, -180.0, 0.0][i % 3]
        p[0][0] = (snap if i % 5 != 2 else 0.0, p[0][0][1])  # a vertex exactly on the antimeridian or prime meridian
        add("antimeridian", [p])
    for i in range(50):
        lo, la = rng.uniform(-180, 180), rng.uniform(-70, 70)
        w = [2.0, 30.0, 95.0, 120.0, 150.0][i % 5]
        kind = i % 10
        if kind < 4:  # an edge along the equator, up to 150 degrees long
            ring = [(lo, 0.0), (lo + w, 0.0), (lo + w / 2, rng.choice([-1, 1]) * rng.uniform(1, 60))]
        elif kind < 7:  # meridional sides
            h = rng.uniform(0.5, 40)
            la = float(np.clip(la, -85 + h, 85 - h))
            ring = [(lo, la), (lo + w / 10, la), (lo + w / 10, la + h), (lo, la + h)]
        else:  # edges longer than 90 degrees
            ring = [(lo, -40.0 + rng.uniform(-5, 5)), (lo + w, 10.0 + rng.uniform(-5, 5)), (lo + w / 3, 50.0 + rng.uniform(-5, 5))]
        if rng.random() < 0.5:
            ring = ring[::-1]
        add("special", [[ring]])
    for i in range(50):
        sgn = 1 if i % 2 else -1
        lo = rng.uniform(-180, 180)
        if i % 4 < 2:  # around a pole, both windings
            k = int(rng.integers(3, 9))
            t = np.sort(rng.uniform(0, 360, k))
            la = sgn * rng.uniform(60, 89.9)
            ring = [(float(lo + x), float(la + rng.uniform(-0.05, 0.05))) for x in t]
        else:  # a vertex on the pole
            la = sgn * rng.uniform(0, 80)
            ring = [(float(lo), sgn * 90.0), (float(lo + rng.uniform(-60, 60)), la), (float(lo + rng.uniform(-60, 60)), la + rng.uniform(-5, 5))]
        if rng.random() < 0.5:
            ring = ring[::-1]
        add("pole", [[ring]])
    for i in range(30):
        if i < 20:  # larger than a hemisphere: a ring south of the equator taken counter-clockwise around the north pole
            k = int(rng.integers(4, 9))
            t = np.sort(rng.uniform(0, 360, k))
            la = rng.uniform(-40, -1)
            ring = [(float(x - 180), float(la + rng.uniform(-2, 2))) for x in t]
        else:  # a near-antipodal edge
            la = rng.uniform(-40, 40)
            lo = rng.uniform(-180, 180)
            ring = [(lo, la), (lo + 179.5 + rng.uniform(-0.4, 0.4), -la + rng.uniform(-0.3, 0.3)), (lo + 90, rng.uniform(-10, 10))]
        if rng.random() < 0.3:
            ring = ring[::-1]
        add("large", [[ring]])
    return rows


def _pair_task(p):
    s, a1, a2, lam, e = T.inverse(*p, with_area=True)
    hav, _ = T.haversine(*p)
    return [T.split(v) for v in (s, a1, a2, lam, e, hav)]


def _ring_task(coords):
    return T.ring(coords)[2]  # [(s, E, dlambda)] mpf


@T._at_dps
def build():
    pairs, pfam = make_pairs()
    polys = make_polygons()
    ring_list = [ring for _, _, ps in polys for p in ps for ring in p]
    with multiprocessing.Pool(os.cpu_count()) as pool:
        pt = pool.map(_pair_task, [tuple(r) for r in pairs], chunksize=4)
        edges = pool.map(_ring_task, ring_list, chunksize=1)
    out = {"pair_in": pairs, "pair_family": pfam}
    for j, name in enumerate(["s12", "alp1", "alp2", "lam12", "E12", "haversine"]):
        out["pair_" + name] = np.array([r[j] for r in pt], dtype=np.float64)
    # polygons: flattened rings, rings per polygon, polygons per row, and the per-edge truths the rows sum
    xy, ring_off, part_off, row_off, edge_off, edge = [], [0], [0], [0], [0], []
    fam, multi, sa, ua, per = [], [], [], [], []
    k = 0
    for f, m, ps in polys:
        fam.append(f)
        multi.append(m)
        sig, uns, perim = T.mp.mpf(0), T.mp.mpf(0), T.mp.mpf(0)
        for p in ps:
            rs_s, rs_u = [], []
            for ri, ring in enumerate(p):
                xy.extend(ring)
                ring_off.append(len(xy))
                e = edges[k]
                k += 1
                edge.extend([(T.split(s), T.split(a), T.split(d)) for s, a, d in e])
                edge_off.append(len(edge))
                rs_s.append(T.ring_from_edges(e, reverse=ri > 0, signed=True))
                rs_u.append(T.ring_from_edges(e, reverse=ri > 0, signed=False))
            part_off.append(len(ring_off) - 1)
            a_s, pp = T.polygon_from_rings(rs_s)
            a_u, _ = T.polygon_from_rings(rs_u)
            sig, uns, perim = sig + a_s, uns + a_u, perim + pp
        row_off.append(len(part_off) - 1)
        sa.append(T.split(sig))
        ua.append(T.split(uns))
        per.append(T.split(perim))
    out.update(poly_xy=np.array(xy, dtype=np.float64), poly_ring_off=np.array(ring_off, dtype=np.int64),
               poly_part_off=np.array(part_off, dtype=np.int64), poly_row_off=np.array(row_off, dtype=np.int64),
               poly_family=np.array(fam, dtype=np.int8), poly_multi=np.array(multi, dtype=bool),
               poly_area_signed=np.array(sa), poly_area_unsigned=np.array(ua), poly_perimeter=np.array(per),
               poly_edge_off=np.array(edge_off, dtype=np.int64), poly_edge=np.array(edge, dtype=np.float64))
    return out


def write(path, arrays):
    with zipfile.ZipFile(path, "w", zipfile.ZIP_STORED) as z:
        for name in sorted(arrays):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.ascontiguousarray(arrays[name]), allow_pickle=False)
            z.writestr(zipfile.ZipInfo(name + ".npy", date_time=(1980, 1, 1, 0, 0, 0)), buf.getvalue())


if __name__ == "__main__":
    write(sys.argv[1] if len(sys.argv) > 1 else OUT, build())
