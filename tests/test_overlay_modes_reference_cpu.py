"""The overlay-modes referees (overlay_modes_reference.py) on their own: exact rings of hand cases, a remainder that does not
depend on the order of the cutters, the exact area identities area(A △ B) = area(A) + area(B) - 2 area(A ∩ B) and
area(s) = area(remainder) + area(s ∩ ∪C), and valid output."""
import itertools
import random
from fractions import Fraction as F

import pytest

import boolean_reference as br
import dissolve_reference as dr
import overlay_modes_reference as omr
import overlay_reference as ov
import validity_reference as vr
from test_overlay_area_model import case_pairs


def _exact(members):
    return [[[(F(x), F(y)) for x, y in r] for r in m] for m in members]


def _valid(members):
    return vr.validity_code("multipolygon", br.as_float(members)) == 0


@pytest.mark.parametrize("k", range(len(omr.symmetric_difference_hand_cases())))
def test_symmetric_difference_hand_cases(k):
    a, b, want = omr.symmetric_difference_hand_cases()[k]
    got = omr.symmetric_difference(a, b)
    assert got == _exact(want), br.as_float(got)
    assert omr.symmetric_difference(b, a) == got
    assert _valid(got)


@pytest.mark.parametrize("k", range(len(omr.remainder_hand_cases())))
def test_remainder_hand_cases_in_every_cutter_order(k):
    s, cutters, want = omr.remainder_hand_cases()[k]
    got = omr.remainder(s, cutters)
    for perm in itertools.permutations(cutters):
        assert omr.remainder(s, list(perm)) == got
    if want is not None:
        assert got == _exact(want), br.as_float(got)
    assert _valid(got)
    cover = dr.union_all(cutters)
    assert ov.polygon_area(s) == br.area(got) + br.area(br.boolean_op(s, cover, "intersection"))


@pytest.mark.parametrize("start", range(0, 120, 10))
def test_symmetric_difference_area_identity_on_model_pairs(start):
    for a, b in case_pairs(40)[start:start + 10]:
        got = omr.symmetric_difference(a, b)
        assert br.area(got) == ov.polygon_area(a) + ov.polygon_area(b) - 2 * ov.intersection_area(a, b)
        assert _valid(got)


@pytest.mark.parametrize("start", range(0, 120, 20))
def test_remainder_area_identity_and_order_on_model_groups(start):
    pairs = case_pairs(40)[start:start + 20]
    rng = random.Random(start)
    for k in range(0, len(pairs) - 3, 4):
        s = pairs[k][0]
        cutters = [pairs[k + t][1] for t in range(4)]
        got = omr.remainder(s, cutters)
        perm = cutters[:]
        rng.shuffle(perm)
        assert omr.remainder(s, perm) == got
        cover = dr.union_all(cutters)
        assert ov.polygon_area(s) == br.area(got) + br.area(br.boolean_op(s, cover, "intersection"))
        assert _valid(got)
