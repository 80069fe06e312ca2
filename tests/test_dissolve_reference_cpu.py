"""The dissolve referee (dissolve_reference.py) on its own: an exact union does not depend on the order of the rows, its area
is inclusion-exclusion of the pairwise intersection areas when no three rows overlap, its output is valid, and the hand
groups give their exact rings."""
import random
from fractions import Fraction as F

import pytest

import boolean_reference as br
import dissolve_reference as dr
import overlay_reference as ov
import validity_reference as vr
from test_overlay_area_model import case_pairs


def _normal(members):
    return [[[(F(x), F(y)) for x, y in r] for r in m] for m in members]


@pytest.mark.parametrize("case", range(len(dr.hand_groups())))
def test_hand_groups_every_order(case):
    rows, want = dr.hand_groups()[case]
    got = dr.union_all(rows)
    rng = random.Random(case)
    for _ in range(12):  # random orders of all the rows, and the reversed order
        perm = rows[:]
        rng.shuffle(perm)
        assert dr.union_all(perm) == got
    assert dr.union_all(rows[::-1]) == got
    if want is not None:
        assert got == _normal(want), br.as_float(got)
    assert vr.validity_code("multipolygon", br.as_float(got)) == 0


def _area(members):
    return ov.polygon_area(members)


@pytest.mark.parametrize("start", range(0, 120, 10))
def test_area_is_inclusion_exclusion_on_model_pairs(start):
    pairs = case_pairs(40)[start:start + 10]
    for a, b in pairs:
        rows = [a, b, dr.row(dr.sq(100, 100, 1))]  # a third, disjoint row: no triple overlap
        got = dr.union_all(rows)
        want = _area(a) + _area(b) + 1 - ov.intersection_area(a, b)
        assert br.area(got) == want
        assert dr.union_all(rows[::-1]) == got
        assert vr.validity_code("multipolygon", br.as_float(got)) == 0


def test_dissolve_groups_and_skips():
    rows = [dr.row(dr.sq(0, 0, 1)), None, dr.row(dr.sq(1, 0, 1)), dr.row(dr.sq(5, 5, 1))]
    out = dr.dissolve(rows, [0, 0, 0, -1], 2)
    assert out[0] == _normal([[[(0, 0), (1, 0), (2, 0), (2, 1), (1, 1), (0, 1), (0, 0)]]])
    assert out[1] == []
