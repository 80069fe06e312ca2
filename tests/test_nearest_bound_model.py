"""CPU model of the pruning bounds of the nearest join (k_nearest.cu, DESIGN.md §4.12), restated in Python doubles.

The kernel drops a right row j for a point p when lb_j > U + tau, where lb_j is the distance from p to the box of all
of j's coordinates, U an upper bound of the answer and tau = 2^-40 * max(M, |px|, |py|) (M: largest absolute
coordinate of the grid's union box).  That is safe only if the computed distance never falls below lb_j - tau, and
if the window bound (the distance to the cells not yet searched) never exceeds the true distance by more than tau.
Distances use glibc's hypot through ctypes, which is what gpl_hypot reproduces bit for bit (Python's math.hypot is a
different algorithm); lb is inflated by 2 ulp because the kernel computes it with CUDA's hypot (<= 2 ulp)."""
import ctypes
import ctypes.util
import math

import numpy as np

_libm = ctypes.CDLL(ctypes.util.find_library("m") or "libm.so.6")
_libm.hypot.restype = ctypes.c_double
_libm.hypot.argtypes = [ctypes.c_double, ctypes.c_double]
hypot = _libm.hypot
EPS = 2.220446049250313e-16


def pt_dist(p, q):
    return hypot(q[0] - p[0], q[1] - p[1])


def line_segment_distance(p, s, e):
    """common.cuh line_segment_distance, operation for operation"""
    if s[0] == e[0] and s[1] == e[1]:
        return pt_dist(p, s)
    dx, dy = e[0] - s[0], e[1] - s[1]
    d2 = dx * dx + dy * dy
    r = ((p[0] - s[0]) * dx + (p[1] - s[1]) * dy) / d2
    if r <= 0.0:
        return pt_dist(p, s)
    if r >= 1.0:
        return pt_dist(p, e)
    sv = ((s[1] - p[1]) * dx - (s[0] - p[0]) * dy) / d2
    return abs(sv) * hypot(dx, dy)


def ls_contains(pts, p):
    """point_dist.cuh line_string_contains_point for n >= 2 (geo's epsilon rule)"""
    for q in pts:
        if q[0] == p[0] and q[1] == p[1]:
            return True
    for s, e in zip(pts[:-1], pts[1:]):
        dx, dy = e[0] - s[0], e[1] - s[1]
        hx, hy = dx != 0.0, dy != 0.0
        tx = (p[0] - s[0]) / dx if hx else 0.0
        ty = (p[1] - s[1]) / dy if hy else 0.0
        if not hx and not hy:
            c = p[0] == s[0] and p[1] == s[1]
        elif hx and not hy:
            c = p[1] == s[1] and 0.0 <= tx <= 1.0
        elif not hx and hy:
            c = p[0] == s[0] and 0.0 <= ty <= 1.0
        else:
            c = abs(tx - ty) <= EPS and 0.0 <= tx <= 1.0
        if c:
            return True
    return False


def point_ls_distance(pts, p):
    if ls_contains(pts, p):
        return 0.0
    return min(line_segment_distance(p, s, e) for s, e in zip(pts[:-1], pts[1:]))


def box_of(pts):
    a = np.asarray(pts)
    return a[:, 0].min(), a[:, 1].min(), a[:, 0].max(), a[:, 1].max()


def lb(p, box):
    x0, y0, x1, y1 = box
    v = hypot(max(max(x0 - p[0], p[0] - x1), 0.0), max(max(y0 - p[1], p[1] - y1), 0.0))
    return math.nextafter(math.nextafter(v, math.inf), math.inf)  # CUDA hypot: up to 2 ulp above glibc's


def tau(M, p, scale=2.0 ** -40):
    return scale * max(M, abs(p[0]), abs(p[1]))


def adversarial(rng):
    """(linestring, point) pairs: 1e6 offsets, 1e-10 extents, long near-axis segments, points on box edges and near
    vertices, lattice input"""
    for _ in range(4000):
        kind = rng.integers(6)
        if kind == 0:  # nybb-like: 1e6 offsets, metre-scale geometry
            o = rng.uniform(9e5, 1.1e6, 2)
            pts = [tuple(o + rng.uniform(-500, 500, 2)) for _ in range(int(rng.integers(2, 6)))]
            p = tuple(o + rng.uniform(-800, 800, 2))
        elif kind == 1:  # 1e-10 extents far from the origin
            o = rng.uniform(-1e3, 1e3, 2)
            pts = [tuple(o + rng.uniform(0, 1e-10, 2)) for _ in range(3)]
            p = tuple(o + rng.uniform(-2e-10, 3e-10, 2))
        elif kind == 2:  # long near-axis segment, point just off it (the cross product cancels)
            L = 10.0 ** rng.uniform(0, 7)
            s = (rng.uniform(-L, L), rng.uniform(-1, 1))
            e = (s[0] + L * rng.choice([-1, 1]), s[1] + rng.uniform(-1e-9, 1e-9) * L)
            pts = [s, e]
            t = rng.uniform(0, 1)
            p = (s[0] + t * (e[0] - s[0]), s[1] + rng.choice([-1, 1]) * 10.0 ** rng.uniform(-12, 1))
        elif kind == 3:  # point on an edge of the box
            pts = [tuple(rng.uniform(-50, 50, 2)) for _ in range(int(rng.integers(2, 5)))]
            x0, y0, x1, y1 = box_of(pts)
            p = (rng.choice([x0, x1]), rng.uniform(y0 - 1, y1 + 1)) if rng.integers(2) else (rng.uniform(x0 - 1, x1 + 1), rng.choice([y0, y1]))
        elif kind == 4:  # near a vertex / on a segment by the epsilon rule
            pts = [tuple(rng.uniform(-50, 50, 2)) for _ in range(3)]
            t = rng.uniform(0, 1)
            p = (pts[0][0] + t * (pts[1][0] - pts[0][0]), pts[0][1] + t * (pts[1][1] - pts[0][1]))
        else:  # lattice
            pts = [tuple(np.round(rng.uniform(0, 10, 2), 1)) for _ in range(int(rng.integers(2, 5)))]
            p = tuple(np.round(rng.uniform(-1, 11, 2), 1))
        yield pts, p


def test_computed_distance_never_below_lb_minus_tau():
    rng = np.random.default_rng(0)
    worst = 0.0
    for pts, p in adversarial(rng):
        box = box_of(pts)
        M = max(abs(v) for v in box)
        d = point_ls_distance(pts, p)
        t = tau(M, p)
        assert d >= lb(p, box) - t, (pts, p)
        if t > 0:
            worst = max(worst, (lb(p, box) - d) / t)
    assert worst < 2.0 ** -6  # the slack is used to well under 2 % of tau


def test_issue_example_needs_the_slack():
    """(0.5, 1) against (0, 0)-(49, 0): the computed distance is 1 ulp below the exact box distance 1"""
    d = line_segment_distance((0.5, 1.0), (0.0, 0.0), (49.0, 0.0))
    assert d == 0.9999999999999999 and d < 1.0 == hypot(0.0, 1.0)
    assert d >= 1.0 - tau(49.0, (0.5, 1.0))


def jg_cell(v, lo, inv, g):
    t = (v - lo) * inv
    return min(max(math.floor(t), 0), g - 1) if math.isfinite(t) else (g - 1 if t > 0 else 0)


def test_window_bound_covers_the_cell_rounding():
    """a coordinate mapped to cell >= k lies at or above X(k) - tau/4; one mapped to cell <= k-1 below X(k) + tau/4
    (X(k) = x0 + k * (w / G) as the kernel computes it); a box without width has inv = 0 and one column"""
    rng = np.random.default_rng(1)
    for _ in range(3000):
        x0 = rng.choice([0.0, rng.uniform(-1e6, 1e6), rng.uniform(-1, 1) * 10.0 ** rng.integers(-10, 7)])
        w = rng.choice([0.0, 10.0 ** rng.uniform(-10, 7)])
        g = int(rng.integers(1, 2049))
        x1 = x0 + w
        w = x1 - x0
        inv = g / w if (w > 0 and math.isfinite(g / w)) else 0.0
        M = max(abs(x0), abs(x1))
        small = tau(M, (0.0, 0.0)) / 4
        cw = w / g
        for v in np.concatenate([rng.uniform(x0, x1, 20), [x0, x1], [x0 + k * cw for k in rng.integers(0, g + 1, 10)]]):
            v = min(max(float(v), x0), x1)
            c = jg_cell(v, x0, inv, g)
            if inv == 0.0:
                assert c == 0
                continue
            assert v >= x0 + c * cw - small
            assert v < x0 + (c + 1) * cw + small or c == g - 1


def model_search(rows, p, maxd, G, slack_scale=2.0 ** -40, stop_early=False):
    """the kernel's per-point search (ring search for U, candidates lb <= U + tau from the one designated cell), over
    linestring rows; returns (min distance, sorted tied rows) or (None, [])"""
    boxes = [box_of(r) for r in rows]
    ux0, uy0 = min(b[0] for b in boxes), min(b[1] for b in boxes)
    ux1, uy1 = max(b[2] for b in boxes), max(b[3] for b in boxes)
    w, h = ux1 - ux0, uy1 - uy0
    iw = G / w if w > 0 and math.isfinite(G / w) else 0.0
    ih = G / h if h > 0 and math.isfinite(G / h) else 0.0
    gx, gy = (1 if iw == 0 else G), (1 if ih == 0 else G)
    cw, ch = w / G, h / G
    cells = {}
    for j, b in enumerate(boxes):
        for cy in range(jg_cell(b[1], uy0, ih, G), jg_cell(b[3], uy0, ih, G) + 1):
            for cx in range(jg_cell(b[0], ux0, iw, G), jg_cell(b[2], ux0, iw, G) + 1):
                cells.setdefault((cx, cy), []).append(j)
    M = max(abs(ux0), abs(uy0), abs(ux1), abs(uy1))
    t = slack_scale * max(M, abs(p[0]), abs(p[1]))
    cxp, cyp = jg_cell(p[0], ux0, iw, G), jg_cell(p[1], uy0, ih, G)

    def ring(r):
        for cy in range(max(cyp - r, 0), min(cyp + r, gy - 1) + 1):
            for cx in range(max(cxp - r, 0), min(cxp + r, gx - 1) + 1):
                if max(abs(cx - cxp), abs(cy - cyp)) == r:
                    yield cx, cy

    def bdist(x0, y0, x1, y1):
        return hypot(max(max(x0 - p[0], p[0] - x1), 0.0), max(max(y0 - p[1], p[1] - y1), 0.0))

    U, r = maxd, 0
    while True:
        for c in ring(r):
            for j in cells.get(c, []):
                U = min(U, pt_dist(p, rows[j][0]) + t)
        B, more = math.inf, False
        if cxp + r + 1 < gx:
            more, B = True, min(B, bdist(ux0 + (cxp + r + 1) * cw, uy0, ux1, uy1))
        if cxp - r - 1 >= 0:
            more, B = True, min(B, bdist(ux0, uy0, ux0 + (cxp - r) * cw, uy1))
        if cyp + r + 1 < gy:
            more, B = True, min(B, bdist(ux0, uy0 + (cyp + r + 1) * ch, ux1, uy1))
        if cyp - r - 1 >= 0:
            more, B = True, min(B, bdist(ux0, uy0, ux1, uy0 + (cyp - r) * ch))
        if not more or B - 2 * t > U:
            break
        r += 1
    rs = max(r - 1, 0) if stop_early else r
    cand = []
    for rr in range(rs + 1):
        for cx, cy in ring(rr):
            for j in cells.get((cx, cy), []):
                b = boxes[j]
                if bdist(*b) <= U + t and jg_cell(min(max(p[0], b[0]), b[2]), ux0, iw, G) == cx and jg_cell(min(max(p[1], b[1]), b[3]), uy0, ih, G) == cy:
                    cand.append(j)
    assert len(cand) == len(set(cand))  # each row from one cell only
    d = {j: point_ls_distance(rows[j], p) for j in cand}
    d = {j: v for j, v in d.items() if v <= maxd}
    if not d:
        return None, []
    best = min(d.values())
    return best, sorted(j for j, v in d.items() if v == best)


def brute(rows, p, maxd):
    d = [point_ls_distance(r, p) for r in rows]
    ok = [j for j in range(len(rows)) if d[j] <= maxd]
    if not ok:
        return None, []
    best = min(d[j] for j in ok)
    return best, [j for j in ok if d[j] == best]


def test_model_search_equals_brute_force():
    rng = np.random.default_rng(2)
    for trial in range(60):
        span = 10.0 ** rng.uniform(-3, 6)
        off = rng.uniform(-1e6, 1e6, 2) * (trial % 3 == 0)
        flat = trial % 7 == 0
        rows = []
        for _ in range(int(rng.integers(1, 60))):
            a = off + rng.uniform(0, span, 2)
            b = a + rng.uniform(-span / 5, span / 5, 2)
            if flat:
                a[1] = b[1] = off[1]
            rows.append([tuple(np.round(a, 2)), tuple(np.round(b, 2))])
        G = int(math.ceil(math.sqrt(len(rows))))
        for _ in range(15):
            p = tuple(off + rng.uniform(-0.3 * span, 1.3 * span, 2))
            maxd = [math.inf, span / 10, 0.0][int(rng.integers(3))]
            assert model_search(rows, p, maxd, G) == brute(rows, p, maxd)


def test_negative_controls():
    """with tau = 0 a seeded search finds an input that loses its true nearest row; stopping one ring early loses rows"""
    rng = np.random.default_rng(3)
    lost = None
    for _ in range(20000):
        L = 10.0 ** rng.uniform(0, 3)
        s = (0.0, 0.0)
        e = (L, 0.0)
        p = (rng.uniform(0.1, L - 0.1), 10.0 ** rng.uniform(-1, 1))
        dA = line_segment_distance(p, s, e)
        lbA = hypot(0.0, p[1])
        if dA < lbA:
            # a point row B just beyond A: the true nearest is A
            dB = math.nextafter(dA, math.inf)
            q = (p[0] - dB, p[1])  # at distance dB from p (computed exactly as pt_dist)
            if pt_dist(p, q) != dB or pt_dist(p, q) >= lbA:
                continue
            rows = [[s, e], [q, q]]
            if brute(rows, p, math.inf)[1] == [0] and model_search(rows, p, math.inf, 2, slack_scale=0.0)[1] != [0]:
                lost = (p, L)
                assert model_search(rows, p, math.inf, 2)[1] == [0]
                break
    assert lost is not None
    early = 0
    for _ in range(200):
        rows = [[tuple(rng.uniform(0, 100, 2))] * 2 for _ in range(100)]
        p = tuple(rng.uniform(0, 100, 2))
        early += model_search(rows, p, math.inf, 10, stop_early=True) != brute(rows, p, math.inf)
    assert early > 0
