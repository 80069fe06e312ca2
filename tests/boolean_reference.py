"""Exact-rational referee of the boolean geometry ops (DESIGN.md §4.19) — TEST INFRASTRUCTURE ONLY.

Built by a route other than the kernel's, on the exact arrangement in fractions.Fraction:
  - pieces: every oriented boundary edge cut at its meetings with the other boundary (oracle.exact._cut_params, the cut
    and classify of overlay_reference); a piece is classified by the exact region position of its rational MIDPOINT, and a
    piece on the other boundary by the direction of the collinear edge it lies on (overlay_reference._same_direction_on);
  - linking: kept pieces meet at rational nodes (dictionary of exact points); at a node with several outgoing pieces the
    one that follows is the first clockwise from the reversed incoming direction, compared on the rational piece
    directions themselves;
  - splitting: every traced ring that visits a node twice is split into the loops between its visits;
  - rings: orientation by the exact shoelace sign; a hole goes to the smallest shell (exact area) whose even-odd ray cast
    contains the midpoint of the hole's first piece (a piece midpoint is never on another output ring).
Output as gpl_boolean_op gives it: closed rings, shells counter-clockwise and holes clockwise, each from its lexicographically
smallest vertex, holes by first vertex, members by their shell's first vertex.  Pure-Python loops: small cases only; valid
(OGC) operands only.
"""
from __future__ import annotations

from fractions import Fraction as F
from functools import cmp_to_key

import overlay_reference as ov
from oracle import exact

OPS = ("intersection", "union", "difference")


def _cross(ax, ay, bx, by):
    return ax * by - ay * bx


def kept_pieces(a_members, b_members, op):
    """the kept pieces (start, end) with rational coordinates, each oriented with the result's interior on its left"""
    am, bm = ov._usable(a_members), ov._usable(b_members)
    ea, eb = ov._oriented_edges(am), ov._oriented_edges(bm)
    out = []
    for u, v in ea:
        for a, b, m in ov._pieces(u, v, eb):
            if a == b:
                continue
            pos = exact._region_pos(m, bm) if eb else 0
            if pos == 1:
                state = "same" if ov._same_direction_on(m, u, v, eb) else "opp"
            else:
                state = ("out", None, "in")[pos]
            if state in {"intersection": ("in", "same"), "union": ("out", "same"), "difference": ("out", "opp")}[op]:
                out.append((a, b))
    for u, v in eb:
        for a, b, m in ov._pieces(u, v, ea):
            if a == b:
                continue
            pos = exact._region_pos(m, am) if ea else 0
            if op == "intersection" and pos == 2:
                out.append((a, b))
            elif op == "union" and pos == 0:
                out.append((a, b))
            elif op == "difference" and pos == 2:
                out.append((b, a))
    return out


def _half(rx, ry, dx, dy):
    """0: d strictly left of r, 1: opposite to r, 2: strictly right, 3: along r"""
    c = _cross(rx, ry, dx, dy)
    if c > 0:
        return 0
    if c < 0:
        return 2
    return 1 if rx * dx + ry * dy < 0 else 3


def _link(pieces):
    out_at = {}
    for i, (a, _) in enumerate(pieces):
        out_at.setdefault(a, []).append(i)
    nxt = []
    for a, b in pieces:
        cands = out_at.get(b, [])
        if len(cands) <= 1:
            nxt.append(cands[0] if cands else None)
            continue
        rx, ry = a[0] - b[0], a[1] - b[1]

        def cmp(i, j):  # larger counter-clockwise angle from r = earlier clockwise from r
            di = (pieces[i][1][0] - b[0], pieces[i][1][1] - b[1])
            dj = (pieces[j][1][0] - b[0], pieces[j][1][1] - b[1])
            hi, hj = _half(rx, ry, *di), _half(rx, ry, *dj)
            if hi != hj:
                return hi - hj
            c = _cross(dj[0], dj[1], di[0], di[1])
            return (c > 0) - (c < 0)

        nxt.append(max(cands, key=cmp_to_key(cmp)))
    return nxt


def _loops(pieces, nxt):
    seen = [False] * len(pieces)
    loops = []
    for j0 in range(len(pieces)):
        if seen[j0]:
            continue
        stack, pos, cur = [], {}, j0
        while cur is not None and not seen[cur]:
            seen[cur] = True
            node = pieces[cur][0]
            if node in pos:
                i0 = pos[node]
                loops.append(stack[i0:])
                for k in stack[i0:]:
                    pos.pop(pieces[k][0], None)
                del stack[i0:]
            pos[node] = len(stack)
            stack.append(cur)
            cur = nxt[cur]
        if cur == j0 and stack:
            loops.append(stack)
    return [[pieces[k][0] for k in lp] for lp in loops]


def _area2(pts):
    return sum(_cross(p[0], p[1], q[0], q[1]) for p, q in zip(pts, pts[1:] + pts[:1]))


def _inside_even_odd(m, pts):
    inside = False
    for s, e in zip(pts, pts[1:] + pts[:1]):
        if (s[1] > m[1]) != (e[1] > m[1]):
            x = s[0] + (m[1] - s[1]) * (e[0] - s[0]) / (e[1] - s[1])
            if x > m[0]:
                inside = not inside
    return inside


def _rotate(pts):
    k = min(range(len(pts)), key=lambda i: pts[i])
    r = pts[k:] + pts[:k]
    return r + [r[0]]


def boolean_op(a_members, b_members, op):
    """the result of `op` as a list of members, each [shell, hole, ...], rings closed lists of (Fraction, Fraction)"""
    pieces = kept_pieces(a_members, b_members, op)
    loops = []
    for pts in _loops(pieces, _link(pieces)):
        merged = [p for i, p in enumerate(pts) if p != pts[i - 1]]
        if len(merged) >= 3 and _area2(merged) != 0:
            loops.append(merged)
    shells = [p for p in loops if _area2(p) > 0]
    holes = [p for p in loops if _area2(p) < 0]
    members = [[s] for s in shells]
    for h in holes:
        m = ((h[0][0] + h[1][0]) / 2, (h[0][1] + h[1][1]) / 2)
        best = None
        for k, s in enumerate(shells):
            if _inside_even_odd(m, s) and (best is None or _area2(s) < _area2(shells[best])):
                best = k
        if best is not None:
            members[best].append(h)
    out = []
    for m in members:
        rings = [_rotate(m[0])] + sorted(_rotate(h) for h in m[1:])
        out.append(rings)
    return sorted(out, key=lambda m: m[0][0])


def area(members) -> F:
    return sum(_area2(m[0][:-1]) / 2 + sum(_area2(h[:-1]) / 2 for h in m[1:]) for m in members) if members else F(0)


def as_float(members):
    return [[[(float(x), float(y)) for x, y in r] for r in m] for m in members]


def _sq(x, y, s):
    return [(x, y), (x + s, y), (x + s, y + s), (x, y + s), (x, y)]


def hand_cases():
    """(A, B, op, expected members): exact rings the referee and the kernel must both give"""
    sq = _sq
    big, hole = sq(0, 0, 10), sq(4, 4, 2)[::-1]
    return [
        ([[sq(0, 0, 2)]], [[sq(1, 1, 2)]], "intersection", [[[(1, 1), (2, 1), (2, 2), (1, 2), (1, 1)]]]),
        ([[sq(0, 0, 2)]], [[sq(1, 1, 2)]], "union", [[[(0, 0), (2, 0), (2, 1), (3, 1), (3, 3), (1, 3), (1, 2), (0, 2), (0, 0)]]]),
        ([[sq(0, 0, 2)]], [[sq(1, 1, 2)]], "difference", [[[(0, 0), (2, 0), (2, 1), (1, 1), (1, 2), (0, 2), (0, 0)]]]),
        # identical polygons: A ∩ A = A ∪ A = A, A − A = ∅
        ([[sq(0, 0, 3)]], [[sq(0, 0, 3)[::-1]]], "intersection", [[sq(0, 0, 3)]]),
        ([[sq(0, 0, 3)]], [[sq(0, 0, 3)]], "union", [[sq(0, 0, 3)]]),
        ([[sq(0, 0, 3)]], [[sq(0, 0, 3)]], "difference", []),
        # shared edge
        ([[sq(0, 0, 1)]], [[sq(1, 0, 1)]], "intersection", []),
        ([[sq(0, 0, 1)]], [[sq(1, 0, 1)]], "union", [[[(0, 0), (1, 0), (2, 0), (2, 1), (1, 1), (0, 1), (0, 0)]]]),
        ([[sq(0, 0, 1)]], [[sq(1, 0, 1)]], "difference", [[sq(0, 0, 1)]]),
        # shared vertex only: union keeps both members, touching at (1, 1)
        ([[sq(0, 0, 1)]], [[sq(1, 1, 1)]], "union", [[sq(0, 0, 1)], [sq(1, 1, 1)]]),
        # a vertex of B on an edge of A
        ([[sq(0, 0, 4)]], [[[(2, 0), (3, -1), (3, 1), (2, 0)]]], "difference",
         [[[(0, 0), (2, 0), (3, 1), (3, 0), (4, 0), (4, 4), (0, 4), (0, 0)]]]),
        # two output members touching at a point
        ([[sq(0, 0, 2)]], [[[(-1, -1), (1, 1), (-1, 3), (-1, -1)]], [[(3, -1), (3, 3), (1, 1), (3, -1)]]], "difference",
         [[[(0, 0), (2, 0), (1, 1), (0, 0)]], [[(0, 2), (1, 1), (2, 2), (0, 2)]]]),
        # an output hole touching its shell
        ([[sq(0, 0, 4)]], [[[(2, 0), (3, 2), (1, 2), (2, 0)]]], "difference",
         [[[(0, 0), (2, 0), (4, 0), (4, 4), (0, 4), (0, 0)], [(1, 2), (3, 2), (2, 0), (1, 2)]]]),
        # a union hole bounded by crossing nodes only: a "#" of two bar shapes
        ([[[(0, 1), (4, 1), (4, 2), (0, 2), (0, 1)]], [[(0, 3), (4, 3), (4, 4), (0, 4), (0, 3)]]],
         [[[(1, 0), (2, 0), (2, 5), (1, 5), (1, 0)]], [[(3, 0), (4.5, 0), (4.5, 5), (3, 5), (3, 0)]]], "union",
         [[[(0, 1), (1, 1), (1, 0), (2, 0), (2, 1), (3, 1), (3, 0), (4.5, 0), (4.5, 5), (3, 5), (3, 4), (2, 4), (2, 5), (1, 5), (1, 4),
            (0, 4), (0, 3), (1, 3), (1, 2), (0, 2), (0, 1)], [(2, 2), (2, 3), (3, 3), (3, 2), (2, 2)]]]),
        # island in lake in island
        ([[big, hole], [sq(4.5, 4.5, 1)]], [[sq(-1, -1, 20)]], "intersection", [[big, hole], [sq(4.5, 4.5, 1)]]),
    ]
