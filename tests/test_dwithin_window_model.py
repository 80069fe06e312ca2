"""CPU model of the window and the pruning of the distance-within join (k_dwithin_pts / k_dwithin_geom, DESIGN.md §4.14),
restated in Python doubles.

A left row with box [lx0, lx1] x [ly0, ly1] walks the cells [cell(lx0 - m), cell(lx1 + m)] x [cell(ly0 - m), cell(ly1 + m)],
m = (D + 2 tau)(1 + 2^-40), and keeps a right row j when lb_j <= D + tau (lb: the box-to-box distance, CUDA hypot) and the
cell is j's designated cell.  Two facts make that exact:
  * every row with lb_j <= D + tau has its designated cell inside the window (checked here on adversarial inputs, with lb
    taken 2 ulp below glibc's hypot, the lowest value CUDA's hypot can return);
  * a row with a computed distance d <= D has lb <= D + tau (the §4.12 / §4.13 bound d >= lb - tau / 2).
Negative controls: without the margin (m = D + tau) a seeded search finds a row with lb <= D + tau whose designated cell lies
outside the window, and with tau = 0 a seeded search finds a pair with d <= D that the candidate test drops."""
import math

import numpy as np

from test_nearest_bound_model import adversarial, box_of, hypot, jg_cell, line_segment_distance, point_ls_distance, tau


def margin(D, t):
    return (D + 2.0 * t) * (1.0 + 2.0 ** -40)


def lb_low(a, b):
    """box-to-box distance, the lowest value CUDA's hypot (<= 2 ulp) can give"""
    v = hypot(max(max(b[0] - a[2], a[0] - b[2]), 0.0), max(max(b[1] - a[3], a[1] - b[3]), 0.0))
    return math.nextafter(math.nextafter(v, 0.0), 0.0)


def designated(i0, i1, l0, l1):
    return i1 if i1 < l0 else (i0 if i0 > l1 else max(i0, l0))


class Grid:
    def __init__(self, ux0, uy0, ux1, uy1, g):
        self.x0, self.y0, self.g = ux0, uy0, g
        w, h = ux1 - ux0, uy1 - uy0
        self.iw = g / w if w > 0 and math.isfinite(g / w) else 0.0
        self.ih = g / h if h > 0 and math.isfinite(g / h) else 0.0
        self.M = max(abs(ux0), abs(uy0), abs(ux1), abs(uy1))

    def cx(self, v):
        return jg_cell(v, self.x0, self.iw, self.g)

    def cy(self, v):
        return jg_cell(v, self.y0, self.ih, self.g)


def window(G, lbox, D, m_of=margin, t=None):
    t = tau(G.M, (max(abs(lbox[0]), abs(lbox[2])), max(abs(lbox[1]), abs(lbox[3])))) if t is None else t
    m = m_of(D, t)
    return t, (G.cx(lbox[0] - m), G.cx(lbox[2] + m), G.cy(lbox[1] - m), G.cy(lbox[3] + m))


def lost_candidates(G, lbox, rboxes, D, m_of=margin, lb_fn=lb_low):
    """right boxes with lb <= D + tau whose designated cell lies outside the window"""
    t, (wx0, wx1, wy0, wy1) = window(G, lbox, D, m_of)
    lcx0, lcx1, lcy0, lcy1 = G.cx(lbox[0]), G.cx(lbox[2]), G.cy(lbox[1]), G.cy(lbox[3])
    out = []
    for k, b in enumerate(rboxes):
        if not lb_fn(lbox, b) <= D + t:
            continue
        dx = designated(G.cx(b[0]), G.cx(b[2]), lcx0, lcx1)
        dy = designated(G.cy(b[1]), G.cy(b[3]), lcy0, lcy1)
        if not (wx0 <= dx <= wx1 and wy0 <= dy <= wy1):
            out.append(k)
    return out


def random_case(rng):
    kind = rng.integers(4)
    if kind == 0:  # nybb-like offsets
        o = rng.uniform(9e5, 1.1e6, 2)
        span, D = 2000.0, 10.0 ** rng.uniform(-3, 3)
    elif kind == 1:  # tiny extents far from the origin
        o = rng.uniform(-1e3, 1e3, 2)
        span, D = 1e-8, 10.0 ** rng.uniform(-12, -8)
    elif kind == 2:  # unit square, D around the cell size
        o = np.zeros(2)
        span, D = 1.0, 10.0 ** rng.uniform(-4, 0)
    else:  # a grid straddling 0 (cell edges near 0 have the finest rounding)
        o = np.full(2, -500.0)
        span, D = 1000.0, float(rng.uniform(0, 400))
    G = Grid(o[0], o[1], o[0] + span, o[1] + span, int(rng.integers(1, 2049)))
    rb = []
    for _ in range(64):
        c = o + rng.uniform(-0.2, 1.2, 2) * span
        e = rng.uniform(0, 0.05, 2) * span * (rng.random(2) < 0.7)
        rb.append((c[0], c[1], c[0] + e[0], c[1] + e[1]))
    c = o + rng.uniform(-0.3, 1.3, 2) * span
    e = rng.uniform(0, 0.02, 2) * span * (rng.random(2) < 0.5)
    lbox = (c[0], c[1], c[0] + e[0], c[1] + e[1])
    # rows at exactly D + tau, one ulp either side, from the left box (the window edge)
    t = tau(G.M, (max(abs(lbox[0]), abs(lbox[2])), max(abs(lbox[1]), abs(lbox[3]))))
    for s in (-1, 1):
        for gap in (D + t, math.nextafter(D + t, 0.0), math.nextafter(D + t, math.inf)):
            x = lbox[0] - gap if s < 0 else lbox[2] + gap
            rb.append((x, lbox[1], x, lbox[3]))
    return G, lbox, rb, D


def test_every_candidate_is_inside_the_window():
    rng = np.random.default_rng(0)
    for _ in range(3000):
        G, lbox, rb, D = random_case(rng)
        assert lost_candidates(G, lbox, rb, D) == [], (lbox, D)


def edge_case(seed=0, tries=200_000):
    """a left point p and a right point q on the same y whose designated cell lies just outside the window when the margin
    is dropped (m = D + tau): the gap p.x - q.x rounds down to D + tau, so lb <= D + tau, while fl(p.x - m) rounds up past
    the cell edge q sits just below.  Grid: the union box [-500, 500]^2 at G = 2 puts a cell edge at x = 0, where the rounding
    of v - x0 makes the edge's resolution ulp(500).  Returns (p, q, D)."""
    rng = np.random.default_rng(seed)
    G = Grid(-500.0, -500.0, 500.0, 500.0, 2)
    qx, hi = -1.0, 0.0  # bisect for the last double of cell 0
    assert G.cx(qx) == 0 and G.cx(hi) == 1
    while math.nextafter(qx, math.inf) != hi:
        mid = qx + (hi - qx) / 2.0
        if mid == qx or mid == hi:
            mid = math.nextafter(qx, math.inf)
        if G.cx(mid) == 0:
            qx = mid
        else:
            hi = mid
    for _ in range(tries):
        px = float(rng.uniform(1.0, 499.0))
        t = tau(G.M, (px, 0.0))
        gap = px - qx  # lb exactly (hypot(a, 0) == |a|)
        D = gap - t
        if not D >= 0.0:
            continue
        lim = D + t
        if not gap <= lim:
            continue
        no_margin = lambda D_, t_: D_ + t_
        if lost_candidates(G, (px, 0.0, px, 0.0), [(qx, 0.0, qx, 0.0)], D, m_of=no_margin, lb_fn=lambda a, b: abs(a[0] - b[2])):
            assert lost_candidates(G, (px, 0.0, px, 0.0), [(qx, 0.0, qx, 0.0)], D, lb_fn=lambda a, b: abs(a[0] - b[2])) == []
            return (px, 0.0), (qx, 0.0), D
    raise AssertionError("no window-edge case found")


def test_negative_control_without_the_margin():
    p, q, D = edge_case()
    assert p[0] - q[0] <= D + tau(500.0, p)


def slack_pair(seed=0):
    """a point p and a segment whose computed distance d is below their box distance lb: with D = d the pair matches, and the
    candidate test lb <= D + tau drops it when tau = 0"""
    rng = np.random.default_rng(seed)
    for _ in range(200_000):
        L = 10.0 ** rng.uniform(1, 3)
        p = (float(rng.uniform(0.1, L - 0.1)), float(10.0 ** rng.uniform(-1, 2)))
        s, e = (0.0, 0.0), (L, 0.0)
        d = line_segment_distance(p, s, e)
        if d < p[1]:
            return p, [s, e], d
    raise AssertionError("no slack case found")


def test_computed_distance_within_D_is_a_candidate():
    rng = np.random.default_rng(2)
    for pts, p in adversarial(rng):
        box = box_of(pts)
        M = max(abs(v) for v in box)
        d = point_ls_distance(pts, p)
        # D = d: the pair matches, so the candidate test must keep it
        assert lb_low((p[0], p[1], p[0], p[1]), box) <= d + tau(M, p), (pts, p)


def test_negative_control_tau_zero():
    p, seg, d = slack_pair()
    box = box_of(seg)
    lbv = hypot(0.0, p[1])  # the exact box distance: p is above the segment's box
    assert d <= d and not lbv <= d + 0.0  # tau = 0 drops a matching pair
    assert lbv <= d + tau(max(abs(v) for v in box), p)
