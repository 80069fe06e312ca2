"""An independent CPU reference of the nearest join, written apart from k_nearest.cu.

`nearest_join(rhs, pts_xy, pts_valid, max_distance, use_grid)` returns (nearest_id int32, distance f64, n_tied int32) with
the join's contract (DESIGN.md §4.12): candidate rows R are non-null, have an envelope and only finite coordinates; the
answer is the minimum distance <= max_distance over R, the lowest row at it and the number of rows at it.  Distances
come from the CPU oracle's row-wise `distance` (oracle/geo_oracle.c, its own restatement of geo's EuclideanDistance),
so this reference shares no arithmetic with the GPU routines.

use_grid = False is brute force over R.  use_grid = True is a ring search with its own design: rows are binned by their
full-coordinate box into a uniform grid of its own; the search grows square windows until the region outside the
window lies further than the best upper bound plus a slack tau' = 2^-30 * scale; the upper bound of a row is the
distance to the FARTHEST corner of its box (every point of the row lies in the box); candidates are de-duplicated with a
set; rows whose distance no box bounds (an empty member, a ring or linestring with fewer than two coordinates) are
always candidates.  Both arms must agree bit for bit."""
import math

import numpy as np

from oracle import oracle as og

POINT, LINESTRING, POLYGON, MULTIPOINT, MULTILINESTRING, MULTIPOLYGON = og.POINT, og.LINESTRING, og.POLYGON, og.MULTIPOINT, og.MULTILINESTRING, og.MULTIPOLYGON


def _levels(a):
    """offset levels from rows down to coordinates"""
    t = a.type
    if t == POINT:
        return []
    if t in (LINESTRING, MULTIPOINT):
        return [a.geom_off]
    if t in (POLYGON, MULTILINESTRING):
        return [a.geom_off, a.ring_off]
    return [a.geom_off, a.part_off, a.ring_off]


def _ranges(a):
    """[c0, c1) coordinate range of every row, and the per-row flag 'some member / ring has fewer than 2 coordinates'"""
    n = len(a)
    lv = _levels(a)
    if not lv:
        r = np.arange(n)
        return r, r + 1, np.zeros(n, bool)
    lo, hi = np.arange(n), np.arange(n) + 1
    for off in lv:
        lo, hi = off[lo], off[hi]
    odd = np.zeros(n, bool)
    if a.type in (LINESTRING,):
        odd = (a.geom_off[1:] - a.geom_off[:-1]) < 2
    elif a.type in (POLYGON, MULTILINESTRING):
        short = (a.ring_off[1:] - a.ring_off[:-1]) < 2
        empty_row = a.geom_off[1:] == a.geom_off[:-1]
        cs = np.concatenate([[0], np.cumsum(short)])
        odd = (cs[a.geom_off[1:]] - cs[a.geom_off[:-1]] > 0) | (empty_row & (a.type == POLYGON))
    elif a.type == MULTIPOLYGON:
        short = (a.ring_off[1:] - a.ring_off[:-1]) < 2
        cs = np.concatenate([[0], np.cumsum(short)])
        part_bad = (cs[a.part_off[1:]] - cs[a.part_off[:-1]] > 0) | (a.part_off[1:] == a.part_off[:-1])
        ps = np.concatenate([[0], np.cumsum(part_bad)])
        odd = ps[a.geom_off[1:]] - ps[a.geom_off[:-1]] > 0
    return lo, hi, odd


def candidate_rows(a):
    """R mask, the 'unbounded' flag and the full-coordinate boxes (n, 4)"""
    _, env_valid = og.envelope(a)  # the oracle's envelope: no envelope -> never matches
    lo, hi, odd = _ranges(a)
    fin = np.isfinite(a.xy).all(axis=1)
    cf = np.concatenate([[0], np.cumsum(~fin)])
    R = env_valid.astype(bool) & (cf[hi] - cf[lo] == 0) & (hi > lo)
    if a.valid is not None:
        R &= a.valid
    box = np.full((len(a), 4), np.nan)
    for j in np.nonzero(R)[0]:
        c = a.xy[lo[j]:hi[j]]
        box[j] = (c[:, 0].min(), c[:, 1].min(), c[:, 0].max(), c[:, 1].max())
    return R, odd & R, box


def take(a, rows):
    """rows of an OGArray as a new OGArray (all valid)"""
    rows = np.asarray(rows, dtype=np.int64)
    if a.type == POINT:
        return og.OGArray(POINT, a.xy[rows])
    lv = _levels(a)
    new_offs = []
    idx = rows
    for off in lv:
        cnt = off[idx + 1] - off[idx]
        new_offs.append(np.concatenate([[0], np.cumsum(cnt)]).astype(np.int64))
        idx = np.concatenate([np.arange(off[i], off[i + 1]) for i in idx]) if len(idx) else np.zeros(0, np.int64)
    xy = a.xy[idx]
    names = {1: ["geom_off"], 2: ["geom_off", "ring_off"], 3: ["geom_off", "part_off", "ring_off"]}[len(lv)]
    return og.OGArray(a.type, xy, **dict(zip(names, new_offs)))


def _dist(a, rows, p, threads=1):
    if len(rows) == 0:
        return np.zeros(0)
    sub = take(a, rows)
    pts = og.OGArray(POINT, np.tile(np.asarray(p, np.float64), (len(rows), 1)))
    return og.distance_rowwise(pts, sub, threads=threads)


def _reduce(rows, d, maxd):
    ok = d <= maxd
    if not ok.any():
        return -1, math.nan, 0
    best = d[ok].min()
    at = np.sort(np.asarray(rows)[ok & (d == best)])
    return int(at[0]), float(best), len(at)


def _hyp(dx, dy):
    return math.hypot(dx, dy)


def _box_dist(p, x0, y0, x1, y1):
    return _hyp(max(x0 - p[0], 0.0, p[0] - x1), max(y0 - p[1], 0.0, p[1] - y1))


class GridSearch:
    def __init__(self, a, R, odd, box):
        self.a = a
        self.always = np.nonzero(odd)[0]
        rows = np.nonzero(R & ~odd)[0]
        self.rows = rows
        self.box = box
        if len(rows) == 0:
            self.g = 0
            return
        b = box[rows]
        self.x0, self.y0 = b[:, 0].min(), b[:, 1].min()
        self.x1, self.y1 = b[:, 2].max(), b[:, 3].max()
        self.g = max(1, int(math.isqrt(len(rows))))
        self.cw = (self.x1 - self.x0) / self.g
        self.ch = (self.y1 - self.y0) / self.g
        self.scale = max(abs(self.x0), abs(self.y0), abs(self.x1), abs(self.y1))
        cells = {}
        for j, (bx0, by0, bx1, by1) in zip(rows, b):
            for cy in range(self._cy(by0), self._cy(by1) + 1):
                for cx in range(self._cx(bx0), self._cx(bx1) + 1):
                    cells.setdefault((cx, cy), []).append(int(j))
        self.cells = cells

    def _c(self, v, lo, w):
        if w <= 0 or not math.isfinite(self.g / w):
            return 0
        return min(max(int(math.floor((v - lo) / w * self.g)), 0), self.g - 1)

    def _cx(self, v):
        return self._c(v, self.x0, self.x1 - self.x0)

    def _cy(self, v):
        return self._c(v, self.y0, self.y1 - self.y0)

    def query(self, p, maxd):
        cand = set(int(j) for j in self.always)
        if self.g:
            tau = 2.0 ** -30 * max(self.scale, abs(p[0]), abs(p[1]))
            # a cell index may be off by one at a cell edge (rounding): windows are widened by one cell, and the bound
            # below measures the distance to what lies outside the widened window's nominal edges
            cx, cy = self._cx(p[0]), self._cy(p[1])
            U = maxd
            seen = set()
            r = 0
            while True:
                for yy in range(cy - r, cy + r + 1):
                    for xx in range(cx - r, cx + r + 1):
                        for j in self.cells.get((xx, yy), ()):
                            if j not in seen:
                                seen.add(j)
                                bx0, by0, bx1, by1 = self.box[j]
                                far = _hyp(max(abs(p[0] - bx0), abs(p[0] - bx1)), max(abs(p[1] - by0), abs(p[1] - by1)))
                                U = min(U, far + tau)
                # inside the window [cx-r+1, cx+r-1] for sure; outside it the distance is at least
                inner_x0 = self.x0 + (cx - r + 1) * self.cw if cx - r >= 1 else -math.inf
                inner_x1 = self.x0 + (cx + r) * self.cw if cx + r <= self.g - 2 else math.inf
                inner_y0 = self.y0 + (cy - r + 1) * self.ch if cy - r >= 1 else -math.inf
                inner_y1 = self.y0 + (cy + r) * self.ch if cy + r <= self.g - 2 else math.inf
                if self.cw == 0:
                    inner_x0, inner_x1 = -math.inf, math.inf
                if self.ch == 0:
                    inner_y0, inner_y1 = -math.inf, math.inf
                gaps = [p[0] - inner_x0, inner_x1 - p[0], p[1] - inner_y0, inner_y1 - p[1]]
                B = min(gaps)
                if B == math.inf or B - 2 * tau > U:
                    break
                r += 1
            for j in seen:
                if _box_dist(p, *self.box[j]) <= U + tau:
                    cand.add(j)
        rows = np.array(sorted(cand), dtype=np.int64)
        return _reduce(rows, _dist(self.a, rows, p), maxd)


def nearest_join(a, pts_xy, pts_valid=None, max_distance=math.inf, use_grid=False, threads=1):
    """(nearest_id, distance, n_tied) per point, by brute force (use_grid=False) or by the ring search (True)"""
    if not (max_distance >= 0):
        raise ValueError("max_distance must be >= 0 or +inf")
    pts = np.asarray(pts_xy, np.float64).reshape(-1, 2)
    n = len(pts)
    R, odd, box = candidate_rows(a)
    nid = np.full(n, -1, np.int32)
    dist = np.full(n, np.nan)
    tied = np.zeros(n, np.int32)
    rows = np.nonzero(R)[0]
    gs = GridSearch(a, R, odd, box) if use_grid else None
    for i, p in enumerate(pts):
        if (pts_valid is not None and not pts_valid[i]) or not np.isfinite(p).all():
            continue
        if gs is None:
            nid[i], dist[i], tied[i] = _reduce(rows, _dist(a, rows, p, threads), max_distance)
        else:
            nid[i], dist[i], tied[i] = gs.query(p, max_distance)
    return nid, dist, tied


def second_gap_ok(a, p, best, tol=1e-9, R=None):
    """True when the second-best distance over R differs from the best by more than tol (relative)"""
    R = candidate_rows(a)[0] if R is None else R
    pts = og.OGArray(POINT, np.tile(np.asarray(p, np.float64), (len(a), 1)))
    d = np.sort(og.distance_rowwise(pts, a)[R])
    d = d[np.isfinite(d)]
    if len(d) < 2:
        return True
    return abs(d[1] - d[0]) > tol * max(abs(d[0]), abs(d[1]), 1e-300)
