"""Exact-rational referees of the symmetric difference and of the remainders of the overlay modes (DESIGN.md §4.23) — TEST
INFRASTRUCTURE ONLY.

Built by other routes than the kernels', on boolean_reference's exact arrangement in fractions.Fraction:
  - symmetric difference: the union of the two differences, (A - B) ∪ (B - A);
  - remainder of a subject: the fold acc <- acc - c over its cutters, one exact difference at a time, so no crossing point is
    rounded and the order of the cutters cannot matter.
The kernel cuts the subject and all of its cutters at once and classifies each piece against all of them.  Output in the form
gpl_boolean_op gives.  Pure Python: small cases of valid (OGC) rows only.
"""
from __future__ import annotations

import boolean_reference as br


def symmetric_difference(a, b):
    """A △ B as a list of members with Fraction coordinates"""
    return br.boolean_op(br.boolean_op(a, b, "difference"), br.boolean_op(b, a, "difference"), "union")


def remainder(subject, cutters):
    """the subject minus every cutter (lists of members)"""
    acc = br.boolean_op(subject, [], "difference")
    for c in cutters:
        acc = br.boolean_op(acc, c, "difference")
    return acc


def _sq(x, y, s):
    return br._sq(x, y, s)


def _rect(x0, y0, x1, y1):
    return [(x0, y0), (x1, y0), (x1, y1), (x0, y1), (x0, y0)]


def symmetric_difference_hand_cases():
    """(A, B, expected members)"""
    sq = _sq
    return [
        # two overlapping squares: two L-shapes touching at (2, 1) and (1, 2)
        ([[sq(0, 0, 2)]], [[sq(1, 1, 2)]],
         [[[(0, 0), (2, 0), (2, 1), (1, 1), (1, 2), (0, 2), (0, 0)]], [[(1, 2), (2, 2), (2, 1), (3, 1), (3, 3), (1, 3), (1, 2)]]]),
        # a full shared edge and a partial one: one member, the shared edge gone
        ([[sq(0, 0, 1)]], [[sq(1, 0, 1)]], [[[(0, 0), (1, 0), (2, 0), (2, 1), (1, 1), (0, 1), (0, 0)]]]),
        ([[sq(0, 0, 2)]], [[sq(2, 1, 2)]], [[[(0, 0), (2, 0), (2, 1), (4, 1), (4, 3), (2, 3), (2, 2), (0, 2), (0, 0)]]]),
        # identical operands, either orientation: empty
        ([[sq(0, 0, 3)]], [[sq(0, 0, 3)]], []),
        ([[sq(0, 0, 3)]], [[sq(0, 0, 3)[::-1]]], []),
        # one square inside another: a shell with a hole, either way round
        ([[sq(0, 0, 4)]], [[sq(1, 1, 2)]], [[sq(0, 0, 4), sq(1, 1, 2)[::-1]]]),
        ([[sq(1, 1, 2)]], [[sq(0, 0, 4)]], [[sq(0, 0, 4), sq(1, 1, 2)[::-1]]]),
        # disjoint: both
        ([[sq(0, 0, 1)]], [[sq(3, 0, 1)]], [[sq(0, 0, 1)], [sq(3, 0, 1)]]),
    ]


def remainder_hand_cases():
    """(subject, cutters, expected members or None when only the referee's answer is pinned)"""
    sq, rect = _sq, _rect
    s = [[sq(0, 0, 4)]]
    return [
        # a cutter splitting the subject in two
        (s, [[[rect(1, -1, 2, 5)]]], [[rect(0, 0, 1, 4)], [rect(2, 0, 4, 4)]]),
        # two cutters sharing an edge inside the subject: one hole, no edge left at x = 2
        (s, [[[rect(1, 1, 2, 3)]], [[rect(2, 1, 3, 3)]]],
         [[sq(0, 0, 4), [(1, 1), (1, 3), (2, 3), (3, 3), (3, 1), (2, 1), (1, 1)]]]),
        # overlapping cutters and a duplicate cutter (reversed)
        (s, [[[rect(1, 1, 3, 2)]], [[rect(2, 1, 3, 3)]], [[rect(1, 1, 3, 2)[::-1]]]],
         [[sq(0, 0, 4), [(1, 1), (1, 2), (2, 2), (2, 3), (3, 3), (3, 2), (3, 1), (2, 1), (1, 1)]]]),
        # three cutter edges through (2, 2): a horizontal, a vertical and a diagonal
        (s, [[[rect(1, 1, 3, 2)]], [[rect(2, 0.5, 2.5, 3)]], [[[(1.5, 1.5), (2.5, 2.5), (1.5, 2.5), (1.5, 1.5)]]]], None),
        # a cutter touching the subject at one point from outside: an extra vertex only
        (s, [[[[(2, 0), (1, -1), (3, -1), (2, 0)]]]], [[[(0, 0), (2, 0), (4, 0), (4, 4), (0, 4), (0, 0)]]]),
        # a cutter touching the shell at one point from inside: a hole touching the shell
        (s, [[[[(2, 0), (3, 1), (1, 1), (2, 0)]]]],
         [[[(0, 0), (2, 0), (4, 0), (4, 4), (0, 4), (0, 0)], [(1, 1), (3, 1), (2, 0), (1, 1)]]]),
        # the subject inside a cutter's hole: unchanged
        ([[sq(1, 1, 1)]], [[[sq(0, 0, 4), sq(0.5, 0.5, 2)[::-1]]]], [[sq(1, 1, 1)]]),
        # a cutter covering the subject, and a cutter along one of its edges from outside
        (s, [[[sq(-1, -1, 6)]]], []),
        (s, [[[rect(4, 0, 5, 4)]], [[rect(-1, 1, 0, 3)]]], [[[(0, 0), (4, 0), (4, 4), (0, 4), (0, 3), (0, 1), (0, 0)]]]),
        # no cutters
        (s, [], [[sq(0, 0, 4)]]),
    ]
