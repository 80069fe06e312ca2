"""CPU model of the intersection-area kernel (k_overlay.cu, DESIGN.md §4.16), checked against the cut-and-classify
referee (overlay_reference.py).

The model restates the kernel's formula: B is translated by the symbolic δ = (ε, ε²); every ring is used with its
interior on the left (σ = ±1 from the turn at its lexicographically lowest vertex); for each edge x of either side,
λ(x) = [end of x inside the other side] + Σ over crossings (+t at an exit, −t at an entry), where the indicator is the
signed ray-crossing winding sum; area = ½ Σ σ_x · cross(x0 − o, x1 − o) · λ(x).  Signs are exact (perturbed orient2d
with the coordinate-difference tie-breaks); with `exact_t` every quantity is a Fraction and the area must EQUAL the
referee's, otherwise t and the sums are f64 as in the kernel and must agree within the GPU tolerance."""
from fractions import Fraction as F

import numpy as np
import pytest

import overlay_reference as ref
import shapes


def _orient(a, b, c):
    """exact orient2d(a, b, c) (> 0: counter-clockwise)"""
    return (F(b[0]) - F(a[0])) * (F(c[1]) - F(a[1])) - (F(b[1]) - F(a[1])) * (F(c[0]) - F(a[0]))


def _sgn(v):
    return (v > 0) - (v < 0)


def _cmp(a, b):
    return (a > b) - (a < b)


def sgn_edge_vs_pert_point(p, q, s):
    """sign of orient(p, q, s + δ)"""
    o = _orient(p, q, s)
    return _sgn(o) or _cmp(p[1], q[1]) or _cmp(q[0], p[0]), o


def sgn_pert_edge_vs_point(s, g, p):
    """sign of orient(s + δ, g + δ, p)"""
    o = _orient(s, g, p)
    return _sgn(o) or _cmp(g[1], s[1]) or _cmp(s[0], g[0]), o


def ring_sigma(closed, hole):
    pts = closed[:-1]
    n = len(pts)
    i = min(range(n), key=lambda k: pts[k])
    v = pts[i]
    j, k = (i - 1) % n, (i + 1) % n
    for _ in range(n):
        if pts[j] != v:
            break
        j = (j - 1) % n
    for _ in range(n):
        if pts[k] != v:
            break
        k = (k + 1) % n
    s = _sgn(_orient(pts[j], v, pts[k]))
    return -s if hole else s


def edges_of(members):
    out = []
    for rings in members:
        for h, r in enumerate(rings):
            c = [tuple(map(float, p)) for p in r]
            if len(c) >= 2 and c[0] != c[-1]:
                c.append(c[0])
            if len(c) < 4:
                continue
            s = ring_sigma(c, h > 0)
            if s:
                out += [(p, q, s) for p, q in zip(c[:-1], c[1:]) if p != q]
    return out


def model_area(a_members, b_members, exact_t=True):
    ea, eb = edges_of(a_members), edges_of(b_members)
    if not ea or not eb:
        return F(0) if exact_t else 0.0
    first = next(tuple(map(float, r[0])) for rings in a_members for r in rings if len(r))
    num = (lambda v: v) if exact_t else float

    def cross_o(p, q):
        if exact_t:
            return (F(p[0]) - F(first[0])) * (F(q[1]) - F(first[1])) - (F(q[0]) - F(first[0])) * (F(p[1]) - F(first[1]))
        return (p[0] - first[0]) * (q[1] - first[1]) - (q[0] - first[0]) * (p[1] - first[1])

    def boxes(p, q, s, g):
        return not (max(p[0], q[0]) < min(s[0], g[0]) or max(s[0], g[0]) < min(p[0], q[0]) or
                    max(p[1], q[1]) < min(s[1], g[1]) or max(s[1], g[1]) < min(p[1], q[1]))

    total = num(F(0))
    for p, q, se in ea:  # edges of A against B + δ
        wind, cr = 0, num(F(0))
        for s, g, sf in eb:
            straddle = (s[1] < q[1]) != (g[1] < q[1]) and max(s[0], g[0]) >= q[0]
            box = boxes(p, q, s, g)
            if not (straddle or box):
                continue
            sq, oq = sgn_pert_edge_vs_point(s, g, q)
            if straddle:
                wind += sf * ((sq > 0) if s[1] < q[1] else -(sq < 0))
            if box:
                sp, op = sgn_pert_edge_vs_point(s, g, p)
                if sp != sq and sgn_edge_vs_pert_point(p, q, s)[0] != sgn_edge_vs_pert_point(p, q, g)[0]:
                    t = op / (op - oq) if exact_t else float(op) / (float(op) - float(oq))
                    cr += sf * sp * t
        total += se * cross_o(p, q) * (wind + cr)
    for s, g, sf in eb:  # edges of B + δ against A
        wind, cr = 0, num(F(0))
        for p, q, se in ea:
            straddle = (p[1] <= g[1]) != (q[1] <= g[1]) and max(p[0], q[0]) > g[0]
            box = boxes(p, q, s, g)
            if not (straddle or box):
                continue
            sg, og = sgn_edge_vs_pert_point(p, q, g)
            if straddle:
                wind += se * ((sg > 0) if p[1] <= g[1] else -(sg < 0))
            if box:
                ss, os_ = sgn_edge_vs_pert_point(p, q, s)
                if ss != sg and sgn_pert_edge_vs_point(s, g, p)[0] != sgn_pert_edge_vs_point(s, g, q)[0]:
                    u = os_ / (os_ - og) if exact_t else float(os_) / (float(os_) - float(og))
                    cr += se * ss * u
        total += sf * cross_o(s, g) * (wind + cr)
    a = total / 2
    return a if a > 0 else (F(0) if exact_t else 0.0)


def case_pairs(n_random=200):
    """(A, B) member lists: contains_cases and multi_contains_cases in both orders and each paired with itself"""
    rng = np.random.default_rng(20261016)
    A, B = shapes.contains_cases(rng, n_random)
    MA, MB = shapes.multi_contains_cases()
    base = [([a], [b]) for a, b in zip(A, B)] + [(ma, [mb]) for ma, mb in zip(MA, MB)]
    out = []
    for a, b in base:
        out += [(a, b), (b, a), (a, a), (b, b)]
    return out


def known_cases():
    """(A, B, exact area)"""
    sq = shapes.sq
    big, hole = sq(0, 0, 10), sq(4, 4, 2)[::-1]
    left, right = sq(0, 0, 10), sq(10, 10, 10)
    return [
        ([[sq(0, 0, 2)]], [[sq(1, 1, 2)]], F(1)),                     # overlapping squares
        ([[sq(0, 0, 3)]], [[sq(0, 0, 3)]], F(9)),                     # identical
        ([[sq(0, 0, 3)]], [[sq(0, 0, 3)[::-1]]], F(9)),               # identical, opposite orientation
        ([[sq(0, 0, 1)]], [[sq(1, 0, 1)]], F(0)),                     # shared edge
        ([[sq(1, 0, 1)]], [[sq(0, 0, 1)]], F(0)),                     # shared edge, other order
        ([[sq(0, 0, 1)]], [[sq(1, 0, 1)[::-1]]], F(0)),               # shared edge, the other ring clockwise
        ([[big, hole]], [[sq(4, 4, 2)]], F(0)),                       # a polygon against its own hole
        ([[sq(4, 4, 2)]], [[big, hole]], F(0)),
        ([[left], [right]], [[sq(8, 8, 4)]], F(8)),                   # MultiPolygon across its touching corner
        ([[sq(8, 8, 4)]], [[left], [right]], F(8)),
        ([[big, hole]], [[sq(3, 3, 4)]], F(12)),                      # covers the hole
        ([[sq(0, 0, 1)]], [[sq(5, 5, 1)]], F(0)),                     # disjoint
        ([[sq(0, 0, 1)]], [[sq(1, 1, 1)]], F(0)),                     # touching corners
        ([], [[sq(0, 0, 1)]], F(0)),                                  # empty
        ([[[(0, 0), (1, 0), (0, 0)]]], [[sq(0, 0, 1)]], F(0)),        # ring of 3 coordinates contributes nothing
    ]


@pytest.mark.parametrize("a,b,want", known_cases())
def test_known_answers(a, b, want):
    assert ref.intersection_area(a, b) == want
    assert model_area(a, b) == want
    assert model_area(a, b, exact_t=False) == float(want)


def tolerance(a, b):
    pts = np.array([p for m in (a, b) for rings in m for r in rings for p in r], dtype=np.float64).reshape(-1, 2)
    diag = float(np.hypot(*(pts.max(0) - pts.min(0)))) if len(pts) else 0.0
    return 1e-9 * float(ref.polygon_area(a) + ref.polygon_area(b)) + 1e-12 * diag * diag


def test_model_equals_referee_exactly_and_f64_within_tolerance():
    pairs = case_pairs()
    assert len(pairs) > 800
    positive = 0
    for a, b in pairs:
        want = ref.intersection_area(a, b)
        assert model_area(a, b) == want, (a, b)
        got = model_area(a, b, exact_t=False)
        assert got >= 0.0 and abs(got - float(want)) <= tolerance(a, b), (a, b, got, want)
        positive += want > 0
    assert positive > len(pairs) // 2


def test_referee_self_area_is_the_polygon_area():
    for a, _ in case_pairs(20)[::4]:
        assert ref.intersection_area(a, a) == ref.polygon_area(a)
