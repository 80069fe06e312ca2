"""CPU reference of the great-circle joins (DESIGN.md §4.15), of a design independent of the GPU's grid: a scipy cKDTree over
3-D unit vectors finds the candidates inside a widened chord radius 2 sin(delta / 2), and the oracle's haversine (the C
restatement, called on two-point linestrings) decides.  Each tree arm has a brute-force arm it must agree with bit for bit."""
import math

import numpy as np
from scipy.spatial import cKDTree

from oracle import oracle as og

R = 6371008.8


def haversine(P, Q):
    """the oracle's haversine_distance for the rows of two (n, 2) lon/lat arrays, vectorised: the haversine length of the
    two-point linestring (p, q) is 0.0 + d"""
    P, Q = np.asarray(P, np.float64).reshape(-1, 2), np.asarray(Q, np.float64).reshape(-1, 2)
    n = len(P)
    if n == 0:
        return np.zeros(0)
    xy = np.empty((2 * n, 2))
    xy[0::2], xy[1::2] = P, Q
    return og.geodesic_length(og.OGArray(og.LINESTRING, xy, geom_off=np.arange(0, 2 * n + 1, 2, dtype=np.int64)), "haversine", threads=0)


def eligible(P, valid=None):
    P = np.asarray(P, np.float64).reshape(-1, 2)
    with np.errstate(invalid="ignore"):
        ok = (np.abs(P[:, 1]) <= 90.0) & (np.abs(P[:, 0]) <= 360.0)
    return ok if valid is None else ok & np.asarray(valid, bool)


def unit(P):
    lon, lat = np.radians(P[:, 0]), np.radians(P[:, 1])
    return np.stack([np.cos(lat) * np.cos(lon), np.cos(lat) * np.sin(lon), np.sin(lat)], axis=1)


def chord(delta):
    """a chord radius that holds every row within the angle delta, widened for the rounding of the unit vectors and for
    the 1e-8 rad error of a computed distance near the antipode"""
    return 2.0 * math.sin(min(delta + 1e-7, math.pi) / 2.0) * (1.0 + 1e-9) + 1e-12


def _within(p, js, Q, D):
    d = haversine(np.repeat(p[None, :], len(js), axis=0), Q[js])
    keep = d <= D
    return js[keep], d[keep]


def dwithin(L, Rr, D, lvalid=None, rvalid=None, tree=True):
    """per left row: (sorted right rows with d <= D, their distances)"""
    L, Rr = np.asarray(L, np.float64).reshape(-1, 2), np.asarray(Rr, np.float64).reshape(-1, 2)
    le, re = eligible(L, lvalid), eligible(Rr, rvalid)
    rows = np.nonzero(re)[0]
    t = cKDTree(unit(Rr[rows])) if tree and len(rows) else None
    out = []
    for i in range(len(L)):
        if not le[i] or len(rows) == 0:
            out.append((np.zeros(0, np.int64), np.zeros(0)))
            continue
        js = rows if t is None else rows[np.sort(np.asarray(t.query_ball_point(unit(L[i:i + 1])[0], chord(D / R)), dtype=np.int64))]
        out.append(_within(L[i], js, Rr, D))
    return out


def nearest(L, Rr, maxd=math.inf, lvalid=None, rvalid=None, tree=True):
    """(nearest_id, distance, tied rows per left row): the minimum computed distance <= maxd, lowest row, every tie"""
    L, Rr = np.asarray(L, np.float64).reshape(-1, 2), np.asarray(Rr, np.float64).reshape(-1, 2)
    le, re = eligible(L, lvalid), eligible(Rr, rvalid)
    rows = np.nonzero(re)[0]
    t = cKDTree(unit(Rr[rows])) if tree and len(rows) else None
    nid, dist, ties = np.full(len(L), -1, np.int32), np.full(len(L), np.nan), []
    for i in range(len(L)):
        ties.append(np.zeros(0, np.int64))
        if not le[i] or len(rows) == 0:
            continue
        js = rows
        if t is not None:
            c0, _ = t.query(unit(L[i:i + 1])[0])
            js = rows[np.sort(np.asarray(t.query_ball_point(unit(L[i:i + 1])[0], chord(2.0 * math.asin(min(c0 / 2.0, 1.0)))), dtype=np.int64))]
        d = haversine(np.repeat(L[i][None, :], len(js), axis=0), Rr[js])
        if np.all(np.isnan(d)):
            continue
        u = np.nanmin(d)
        if u <= maxd:
            ties[i] = js[d == u]
            nid[i], dist[i] = ties[i][0], u
    return nid, dist, ties
