"""The exact-rational boolean-geometry referee (boolean_reference.py) pinned on the CPU: exact rings of hand cases, and on the
900+ pairs of test_overlay_area_model.case_pairs() exact area identities against overlay_reference.intersection_area and OGC
validity of every output by validity_reference."""
from fractions import Fraction as F

import pytest

import boolean_reference as br
import overlay_reference as ov
import validity_reference as vr
from test_overlay_area_model import case_pairs, known_cases


def _exact(members):
    return [[[(F(x), F(y)) for x, y in r] for r in m] for m in members]


@pytest.mark.parametrize("k", range(len(br.hand_cases())))
def test_hand_cases(k):
    a, b, op, want = br.hand_cases()[k]
    got = br.boolean_op(a, b, op)
    assert got == _exact(want), (op, br.as_float(got))
    assert vr.validity_code("multipolygon", br.as_float(got)) == 0


def test_empty_operands():
    s = br._sq(0, 0, 1)
    assert br.boolean_op([], [[s]], "intersection") == []
    assert br.boolean_op([], [[s]], "union") == _exact([[s]])
    assert br.boolean_op([[s[::-1]]], [], "difference") == _exact([[s]])
    assert br.boolean_op([], [[s]], "difference") == []


def _pairs():
    return case_pairs() + [(a, b) for a, b, _ in known_cases() if a and b]


@pytest.mark.parametrize("op", br.OPS)
def test_area_identities_and_validity_on_the_case_pairs(op):
    pairs = _pairs()
    assert len(pairs) >= 900
    for i, (a, b) in enumerate(pairs):
        got = br.boolean_op(a, b, op)
        inter = ov.intersection_area(a, b)
        aa, ab = ov.polygon_area(a), ov.polygon_area(b)
        want = {"intersection": inter, "union": aa + ab - inter, "difference": aa - inter}[op]
        assert br.area(got) == want, (op, i, a, b)
        for m in got:
            assert br._area2(m[0][:-1]) > 0 and all(br._area2(h[:-1]) < 0 for h in m[1:])
            for r in m:
                assert r[0] == r[-1] and r[0] == min(r)
        assert vr.validity_code("multipolygon", br.as_float(got)) == 0, (op, i, a, b, br.as_float(got))
