"""The families of tests/boolean_families.py against the exact referees, without a GPU: every operand valid, the referees'
area identities exact on BA (origin), BB and BC, BD's closed forms equal to the referee ring for ring for small k, and the
finding pinned — the referee's exact output of BB, rounded to doubles, is invalid on a stated minimum of rows (spikes and
pinches where two crossings round to one point), so a later edit cannot make the family trivial."""
from collections import Counter

import boolean_families as BF
import boolean_reference as br
import overlay_reference as ov
import pairs_families as PF
import validity_reference as vr


def _mem(c):
    return BF.members(c[0], c[1]), BF.members(c[2], c[3])


def test_operands_valid():
    base, moved = BF.family_ba()
    closed, unclosed = BF.family_bc()
    cases = base + [c for v in moved.values() for c in v] + BF.family_bb() + closed + unclosed + BF.family_bd([1, 2, 3])
    for c in cases:
        assert vr.validity_code(c[0], c[1]) == 0 and vr.validity_code(c[2], c[3]) == 0, c[4]


def _identities(cases):
    for c in cases:
        a, b = _mem(c)
        inter = ov.intersection_area(a, b)
        aa, ab = ov.polygon_area(a), ov.polygon_area(b)
        got = {op: br.area(br.boolean_op(a, b, op)) for op in BF.OPS}
        assert got == {"intersection": inter, "union": aa + ab - inter, "difference": aa - inter}, c[4]


def test_identities_ba_origin():
    _identities(BF.family_ba()[0])


def test_identities_bc():
    _identities(BF.family_bc()[0])


def test_identities_bb_and_the_rounding_finding():
    """BB: exact identities, and the referee's output rounded to doubles invalid on at least 600 (row, op) results —
    ring self-intersections (6, a union pinch) and self-intersections (5, a difference spike) among them — at every offset"""
    cases = BF.family_bb()
    codes, offsets = Counter(), set()
    for c in cases:
        a, b = _mem(c)
        inter = ov.intersection_area(a, b)
        aa, ab = ov.polygon_area(a), ov.polygon_area(b)
        want = {"intersection": inter, "union": aa + ab - inter, "difference": aa - inter}
        for op in BF.OPS:
            r = br.boolean_op(a, b, op)
            assert br.area(r) == want[op], (op, c[4])
            code = vr.validity_code("multipolygon", br.as_float(r))
            if code:
                codes[code] += 1
                offsets.add(c[4].rsplit("@", 1)[1].split()[0])
    assert sum(codes.values()) >= 600 and codes[5] >= 100 and codes[6] >= 100, codes
    assert offsets == {str(o) for o in PF.B_OFFSETS}, offsets


def test_bd_closed_forms_equal_the_referee():
    for c in BF.family_bd([1, 2, 3]):
        a, b = _mem(c)
        for op in BF.OPS:
            assert br.boolean_op(a, b, op) == c[5][op], (op, c[4])
        assert ov.intersection_area(a, b) == c[6], c[4]
        assert br.area(c[5]["intersection"]) == c[6]
