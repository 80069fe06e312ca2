"""The validity referee (tests/validity_reference.py) on the known-answer table, and an executable model of k_valid.cu's
algorithm (chunks of 32 edges, per-row grids, edge-pair relations, touch events with the star union-find, symbolic points)
that must give the referee's code on every known answer and on random lattice rows."""
import math
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from oracle.exact import orient_sign  # noqa: E402
from shapes import random_polygon, sq  # noqa: E402
from validity_reference import validity_code  # noqa: E402

NAN, INF = float("nan"), float("inf")
S = sq(0, 0, 10)


def known_answers():
    """(kind, row, code) of the contract's table"""
    o = sq(0, 0, 4)
    cases = [
        ("polygon", [o], 0), ("polygon", [o[:-1]], 0), ("polygon", [o[:2] + o[1:]], 0), ("polygon", [o[::-1]], 0),
        ("polygon", [S, sq(2, 2, 2)], 0),
        ("polygon", [S, [(0, 5), (3, 3), (3, 7), (0, 5)]], 0),
        ("polygon", [S, [(0, 5), (5, 0), (5, 5), (0, 5)]], 4),
        ("polygon", [S, sq(2, 2, 2), sq(4, 4, 2)], 0),
        ("polygon", [S, [(0, 5), (4, 3), (4, 7), (0, 5)], [(4, 5), (7, 3), (10, 5), (7, 7), (4, 5)]], 4),
        ("polygon", [[(0, 0), (2, 2), (2, 0), (0, 2), (0, 0)]], 5),
        ("polygon", [[(0, 0), (4, 0), (2, 2), (4, 4), (0, 4), (2, 2), (0, 0)]], 6),
        ("polygon", [[(0, 0), (4, 0), (4, 4), (2, 0), (0, 4), (0, 0)]], 6),
        ("polygon", [[(0, 0), (4, 0), (4, 2), (6, 2), (4, 2), (4, 4), (0, 4), (0, 0)]], 5),
        ("polygon", [[(0, 0), (1, 0), (2, 0), (0, 0)]], 5),
        ("polygon", [[(0, 0), (1, 1), (0, 0)]], 9), ("polygon", [[(0, 0), (1, 0), (1, 0), (0, 0)]], 9),
        ("polygon", [[(0, 0), (1, 0), (1, 1)]], 0),
        ("polygon", [S, sq(12, 2, 2)], 2), ("polygon", [S, [(10, 5), (12, 4), (12, 6), (10, 5)]], 2),
        ("polygon", [S, sq(8, 2, 4)], 5), ("polygon", [S, S], 5),
        ("polygon", [S, sq(1, 1, 8), sq(3, 3, 2)], 3),
        ("multipolygon", [[sq(0, 0, 1)], [sq(1, 1, 1)]], 0), ("multipolygon", [[sq(0, 0, 1)], [sq(5, 5, 1)]], 0),
        ("multipolygon", [[sq(0, 0, 1)], [sq(1, 0, 1)]], 5), ("multipolygon", [[sq(0, 0, 2)], [sq(1, 1, 2)]], 5),
        ("multipolygon", [[S], [sq(2, 2, 2)]], 7),
        ("multipolygon", [[S, sq(2, 2, 6)], [sq(4, 4, 2)]], 0),
        ("polygon", [[(0, 0), (2, 2), (2, 0), (NAN, 2), (0, 0)]], 10),
        ("polygon", [sq(0, 0, 2), [(5, 5), (7, 7), (7, 5), (5, 7), (5, 5)]], 5),
        ("linestring", [(0, 0), (1, 1)], 0), ("linestring", [(0, 0), (2, 2), (2, 0), (0, 2)], 0), ("linestring", [], 0),
        ("linestring", [(1, 1), (1, 1)], 9), ("linestring", [(0, 0), (NAN, 1)], 10),
        ("point", (1, 2), 0), ("point", (NAN, NAN), 0), ("point", (NAN, 1), 10), ("point", (INF, 0), 10),
        ("polygon", None, None), ("polygon", [], 0), ("multipolygon", [], 0),
    ]
    return cases


def lattice_rows(rng, n):
    """(kind, row) random (Multi)Polygons on a coarse lattice: holes, members disjoint / touching / sharing edges /
    overlapping / nested, planted defects"""
    out = []
    for i in range(n):
        q = int(rng.integers(0, 2))
        k = i % 6
        if k == 0 and i % 12 == 0:
            out.append(("polygon", random_polygon(rng, 6.0, hole=bool(rng.integers(0, 2)), q=q)))
        elif k == 0:  # square holes: nested, touching, outside
            rings = [sq(0, 0, 10)]
            for _ in range(int(rng.integers(0, 3))):
                a, b = (int(v) for v in rng.integers(0, 11, 2))
                rings.append(sq(a, b, 1 + int(rng.integers(0, 6))))
            if rng.integers(0, 2):  # a hole in a hole
                a, b, c, d = (int(v) for v in rng.integers(0, 6, 4))
                rings += [sq(a, b, 5), sq(a + c % 4, b + d % 4, 1 + int(rng.integers(0, 3)))]
            out.append(("polygon", rings))
        elif k == 1:  # a shell with lattice triangle holes: inside, touching the shell or each other, outside, nested
            rings = [sq(0, 0, 6)]
            for _ in range(int(rng.integers(1, 4))):
                t = [(float(v[0]), float(v[1])) for v in rng.integers(0, 8, (3, 2))]
                rings.append(t if rng.integers(0, 2) else t + [t[0]])
            out.append(("polygon", rings))
        elif k == 2:  # members: disjoint, touching, edge-sharing, overlapping or nested squares
            members = []
            for _ in range(int(rng.integers(1, 4))):
                x, y, s = (int(v) for v in rng.integers(0, 5, 3))
                members.append([sq(x, y, 1 + s % 3)])
            out.append(("multipolygon", members))
        elif k == 3:  # random lattice rings (often self-touching or crossing)
            m = int(rng.integers(3, 8))
            ring = [(float(v[0]), float(v[1])) for v in rng.integers(0, 4, (m, 2))]
            out.append(("polygon", [ring]))
        elif k == 4:  # an island in a lake, or beside it in the shell, or touching either
            a, b = (int(v) for v in rng.integers(0, 9, 2))
            out.append(("multipolygon", [[sq(0, 0, 10), sq(2, 2, 6)], [sq(a, b, 1 + int(rng.integers(0, 3)))]]))
        else:
            out.append(("multipolygon", [random_polygon(rng, 6.0, hole=bool(rng.integers(0, 2)), q=q) for _ in range(int(rng.integers(1, 3)))]))
    return out


# ---- the model: k_valid.cu restated ---------------------------------------------------------------------------------------


def _chain(ring):
    """Chain: coordinates with Polygon::new's closing coordinate emulated"""
    pts = [tuple(map(float, p)) for p in ring]
    if len(pts) >= 2 and pts[0] != pts[-1]:
        pts.append(pts[0])
    return pts


def _edge_relation(p, q, r, s):
    if max(p[0], q[0]) < min(r[0], s[0]) or max(r[0], s[0]) < min(p[0], q[0]) or max(p[1], q[1]) < min(r[1], s[1]) or max(r[1], s[1]) < min(p[1], q[1]):
        return 0, None
    o1, o2 = orient_sign(p, q, r), orient_sign(p, q, s)
    if o1 * o2 > 0:
        return 0, None
    if o1 == 0 and o2 == 0:
        ax = p[0] != q[0]
        pp, qq, rr, ss = (v[0] if ax else v[1] for v in (p, q, r, s))
        lo, hi = max(min(pp, qq), min(rr, ss)), min(max(pp, qq), max(rr, ss))
        if lo < hi:
            return 1, None
        if lo > hi:
            return 0, None
        return 2, (p if pp == lo else q)
    o3, o4 = orient_sign(r, s, p), orient_sign(r, s, q)
    if o3 * o4 > 0:
        return 0, None
    if o1 * o2 < 0 and o3 * o4 < 0:
        return 1, None
    return 2, (r if o1 == 0 else s if o2 == 0 else p if o3 == 0 else q)


def _cmp(a, b):
    return (a > b) - (a < b)


def _sym_ring_pos(q, c):
    """sym_point.cuh: 0 outside / 1 boundary / 2 inside for the symbolic point q = (x, v, side) against the chain c"""
    (xx, xy), (vx, vy), side = q

    def cmp_y(cy):
        return _cmp(cy, xy) or -_cmp(vy, xy) or -side * _cmp(vx, xx)

    def cmp_x(cx):
        return _cmp(cx, xx) or -_cmp(vx, xx) or side * _cmp(vy, xy)

    def orient(s, e):
        o = orient_sign(s, e, (xx, xy)) or orient_sign(s, e, (vx, vy))
        if o or not side:
            return o
        d1, d2 = (_cmp(e[0], s[0]), _cmp(vx, xx)) if e[0] != s[0] else (_cmp(e[1], s[1]), _cmp(vy, xy))
        return side * d1 * d2

    def between(b1, b2):
        lo, hi = min(b1, b2), max(b1, b2)
        return cmp_x(lo) <= 0 and cmp_x(hi) >= 0

    if len(c) < 2:
        return 0
    wn = 0
    for s, e in zip(c[:-1], c[1:]):
        cs, ce = cmp_y(s[1]), cmp_y(e[1])
        if cs <= 0:
            if ce >= 0:
                o = orient(s, e)
                if o > 0 and ce != 0:
                    wn += 1
                elif o == 0 and between(s[0], e[0]):
                    return 1
        elif ce <= 0:
            o = orient(s, e)
            if o < 0:
                wn -= 1
            elif o == 0 and between(s[0], e[0]):
                return 1
    return 2 if wn else 0


def _jg_cell(v, lo, inv, g):
    return min(max(math.floor((v - lo) * inv), 0), g - 1)


def model_code(kind, geom):
    if geom is None:
        return None
    if kind in ("point", "multipoint", "linestring", "multilinestring"):
        return validity_code(kind, geom)  # rules 10 and 9 only: k_valid_rows is a direct reading of the contract
    polys = [geom] if kind == "polygon" else geom
    if not all(math.isfinite(c) for poly in polys for ring in poly for p in ring for c in p):
        return 10
    rings = []  # (member, chain)
    for m, poly in enumerate(polys):
        for ring in poly:
            c = _chain(ring)
            if c and sum(c[i] != c[i + 1] for i in range(len(c) - 1)) < 3:
                return 9
            rings.append((m, c))
    first_ring = {}
    for g, (m, _) in enumerate(rings):
        first_ring.setdefault(m, g)
    # chunks, nd ranks
    chunks = []  # (ring, [(edge index, p, q, rank)], box)
    for g, (m, c) in enumerate(rings):
        ne = len(c) - 1 if len(c) >= 2 else 0
        rank, ranks = 0, {}
        for i in range(ne):
            if c[i] != c[i + 1]:
                ranks[i] = rank
                rank += 1
        for k0 in range(0, ne, 32):
            es = [(i, c[i], c[i + 1], ranks[i]) for i in range(k0, min(ne, k0 + 32)) if i in ranks]
            box = None
            if es:
                xs = [v[0] for e in es for v in e[1:3]]
                ys = [v[1] for e in es for v in e[1:3]]
                box = (min(xs), min(ys), max(xs), max(ys))
            chunks.append((g, es, box, rank))
    boxes = [ch[2] for ch in chunks if ch[2]]
    flags = set()
    events = []
    if boxes:
        x0, y0 = min(b[0] for b in boxes), min(b[1] for b in boxes)
        x1, y1 = max(b[2] for b in boxes), max(b[3] for b in boxes)
        G = int(min(1024.0, math.ceil(math.sqrt(len(chunks)))))
        w, h = x1 - x0, y1 - y0
        iw = G / w if w > 0 and math.isfinite(G / w) else 0.0
        ih = G / h if h > 0 and math.isfinite(G / h) else 0.0
        cells = {}
        for k, ch in enumerate(chunks):
            b = ch[2]
            if not b:
                continue
            for cy in range(_jg_cell(b[1], y0, ih, G), _jg_cell(b[3], y0, ih, G) + 1):
                for cx in range(_jg_cell(b[0], x0, iw, G), _jg_cell(b[2], x0, iw, G) + 1):
                    cells.setdefault(cy * G + cx, []).append(k)

        def cell_of(x, y):
            return _jg_cell(y, y0, ih, G) * G + _jg_cell(x, x0, iw, G)

        pairs = []
        for c, lst in cells.items():
            for t, a in enumerate(lst):
                ba = chunks[a][2]
                if cell_of(ba[0], ba[1]) == c:
                    pairs.append((a, a))
                for b in lst[t + 1:]:
                    bb = chunks[b][2]
                    if bb[2] < ba[0] or ba[2] < bb[0] or bb[3] < ba[1] or ba[3] < bb[1]:
                        continue
                    if cell_of(max(ba[0], bb[0]), max(ba[1], bb[1])) == c:
                        pairs.append((a, b))
        for a, b in pairs:
            ga, ea, _, ka = chunks[a]
            gb, eb, _, _ = chunks[b]
            for ia, (_, p, q, ra) in enumerate(ea):
                for jb, (_, r, s, rb) in enumerate(eb):
                    if a == b and jb <= ia:
                        continue
                    rel, w_ = _edge_relation(p, q, r, s)
                    if rel == 1:
                        flags.add(5)
                    elif rel == 2:
                        if ga == gb:
                            d = (rb - ra) % ka
                            if d not in (1, ka - 1):
                                flags.add(6)
                        elif rings[ga][0] == rings[gb][0]:
                            events.append((min(ga, gb), max(ga, gb), w_))
    if 5 in flags:
        return 5
    if 6 in flags:
        return 6
    # touch cycles: star union-find
    parent = list(range(len(rings)))

    def find(x):
        while parent[x] != x:
            x = parent[x]
        return x

    for i, (a, b, w_) in enumerate(events):
        if any(e[2] == w_ and (e[0] < a or (j < i and e[0] == a and e[1] == b)) for j, e in enumerate(events)):
            continue
        x, y = find(a), find(b)
        if x == y:
            flags.add(4)
            break
        parent[max(x, y)] = min(x, y)
    # ring position
    for g, (m, c) in enumerate(rings):
        if not c:
            continue
        i = 0
        while c[i] == c[i + 1]:
            i += 1
        q = (c[i], c[i + 1], 0)
        g0 = first_ring[m]
        members_rings = [h for h, (mm, _) in enumerate(rings) if mm == m]
        if g > g0:
            if not rings[g0][1] or _sym_ring_pos(q, rings[g0][1]) != 2:
                flags.add(2)
            if any(h != g and h != g0 and rings[h][1] and _sym_ring_pos(q, rings[h][1]) == 2 for h in members_rings):
                flags.add(3)
        elif kind == "multipolygon":
            for mj in set(mm for mm, _ in rings):
                if mj == m or not rings[first_ring[mj]][1]:
                    continue
                rj = [h for h, (mm, _) in enumerate(rings) if mm == mj]
                if _sym_ring_pos(q, rings[rj[0]][1]) == 2 and not any(rings[h][1] and _sym_ring_pos(q, rings[h][1]) == 2 for h in rj[1:]):
                    flags.add(7)
    for code in (2, 3, 7, 4):
        if code in flags:
            return code
    return 0


# ---- tests ------------------------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("case", range(len(known_answers())))
def test_referee_known_answers(case):
    kind, row, want = known_answers()[case]
    assert validity_code(kind, row) == want


@pytest.mark.parametrize("case", range(len(known_answers())))
def test_model_known_answers(case):
    kind, row, want = known_answers()[case]
    assert model_code(kind, row) == want


def test_model_equals_referee_on_random_lattice_rows():
    rng = np.random.default_rng(18)
    rows = lattice_rows(rng, 2400)
    codes = {}
    for kind, row in rows:
        want = validity_code(kind, row)
        assert model_code(kind, row) == want, (kind, row, want)
        codes[want] = codes.get(want, 0) + 1
    # the generator reaches every polygon rule
    assert all(codes.get(c, 0) > 0 for c in (0, 2, 3, 4, 5, 6, 7)), codes


def test_model_and_referee_on_a_ring_longer_than_one_chunk():
    n = 100
    ring = [(round(math.cos(2 * math.pi * i / n) * 50, 3), round(math.sin(2 * math.pi * i / n) * 50, 3)) for i in range(n)]
    assert validity_code("polygon", [ring]) == model_code("polygon", [ring]) == 0
    bad = ring[:40] + [(ring[90][0] * 1.1, ring[90][1] * 1.1)] + ring[41:]  # one vertex moved across the ring: crossings
    assert validity_code("polygon", [bad]) == model_code("polygon", [bad]) == 5
