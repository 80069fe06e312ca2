"""Exact-rational referee of dissolve / union_all (DESIGN.md §4.21) — TEST INFRASTRUCTURE ONLY.

Built by another route than the kernel's: the union of a group is folded row by row, acc <- boolean_reference.boolean_op(acc,
row, "union"), everything in fractions.Fraction, so every intermediate result is exact and the fold order cannot matter.
The kernel cuts each row against all of its partners at once and classifies each piece against all of them.  Output in
the form gpl_boolean_op gives (closed rings, shells counter-clockwise, holes clockwise, each from its smallest vertex, holes
by first vertex, members by their shell's first vertex).  Pure Python: small groups of valid (OGC) rows only.
"""
from __future__ import annotations

import boolean_reference as br


def union_all(rows):
    """the union of the rows (lists of members; None rows skipped) as a list of members with Fraction coordinates"""
    acc = []
    for r in rows:
        if r is None:
            continue
        acc = br.boolean_op(acc, r, "union")
    return acc


def dissolve(rows, codes, n_groups):
    """one union per group code in [0, n_groups); code -1 skips a row"""
    return [union_all([r for r, c in zip(rows, codes) if c == g]) for g in range(n_groups)]


def sq(x, y, s):
    return br._sq(x, y, s)


def row(*rings):
    """a row of one member: its shell and holes"""
    return [list(rings)]


def lattice(k, s=1):
    return [row(sq(i * s, j * s, s)) for j in range(k) for i in range(k)]


def hand_groups():
    """(rows, expected members or None when only the referee's answer is pinned): groups whose union has exact rings"""
    k = 3
    boundary = [(i, 0) for i in range(k)] + [(k, j) for j in range(k)] + [(k - i, k) for i in range(k)] + [(0, k - j) for j in range(k)]
    ring8 = [row(sq(i, j, 1)) for j in range(3) for i in range(3) if (i, j) != (1, 1)]
    outer = [(0, 0), (1, 0), (2, 0), (3, 0), (3, 1), (3, 2), (3, 3), (2, 3), (1, 3), (0, 3), (0, 2), (0, 1)]
    return [
        # a k x k lattice of unit squares: one square with every boundary grid point as a vertex
        (lattice(k), [[boundary + [boundary[0]]]]),
        # a checkerboard: members touching at corners
        ([row(sq(0, 0, 1)), row(sq(1, 1, 1)), row(sq(2, 0, 1))], [[sq(0, 0, 1)], [sq(1, 1, 1)], [sq(2, 0, 1)]]),
        # a ring of 8 squares: a square with a square hole
        (ring8, [[outer + [(0, 0)], [(1, 1), (1, 2), (2, 2), (2, 1), (1, 1)]]]),
        # three identical squares (any orientation)
        ([row(sq(0, 0, 2)), row(sq(0, 0, 2)[::-1]), row(sq(0, 0, 2))], [[sq(0, 0, 2)]]),
        # three edges through one point (1, 1): a horizontal, a vertical and a diagonal crossing
        ([row([(0, 0), (2, 0), (2, 1), (0, 1), (0, 0)]), row([(1, 0.5), (2.5, 0.5), (2.5, 1.5), (1, 1.5), (1, 0.5)]),
          row([(0.5, 0.5), (1.5, 1.5), (0.5, 1.75), (0.5, 0.5)])], None),
        # a crossing through a third row's vertex: the horizontal and vertical edges cross at (1, 1), a vertex of the triangle
        ([row([(0, 0), (2, 0), (2, 1), (0, 1), (0, 0)]), row([(1, 0.5), (2.5, 0.5), (2.5, 1.5), (1, 1.5), (1, 0.5)]),
          row([(1, 1), (0.5, 1.75), (0.25, 1.5), (1, 1)])], None),
        # a row inside another's hole, touching it at one point
        ([row(sq(0, 0, 4), sq(1, 1, 2)[::-1]), row([(2, 1), (2.5, 1.5), (1.5, 1.5), (2, 1)])], None),
        # two rows: an edge of one crosses the other's shell edge exactly where the other's hole touches its shell
        ([row(sq(0, 0, 4), [(2, 0), (1, 1), (3, 1), (2, 0)]), row([(2, -1), (5, -1), (5, 0.5), (2, 0.5), (2, -1)])], None),
        # shared edges and a hole closed by a third row
        ([row([(0, 0), (3, 0), (3, 1), (0, 1), (0, 0)]), row([(0, 1), (1, 1), (1, 3), (0, 3), (0, 1)]),
          row([(2, 1), (3, 1), (3, 3), (2, 3), (2, 1)]), row([(1, 2), (2, 2), (2, 3), (1, 3), (1, 2)])], None),
    ]
