"""CPU tests of the exact-rational clip referee (tests/clip_reference.py, DESIGN.md §4.22): the hand cases with their exact
members, and the partition identities on valid lattice line x polygon pairs (pairs_families.family_a)."""
import math
from fractions import Fraction as F

import pytest

import clip_reference as cr
import pairs_families as pf


@pytest.mark.parametrize("case", cr.HAND, ids=[c[0] for c in cr.HAND])
def test_hand_cases(case):
    name, ka, a, kb, b, want_i, want_d = case
    if ka in ("point", "multipoint"):
        assert cr.clip(ka, a, kb, b) == want_i
        assert cr.clip(ka, a, kb, b, invert=True) == want_d
        return
    assert cr.plain(cr.clip(ka, a, kb, b)) == want_i
    assert cr.plain(cr.clip(ka, a, kb, b, invert=True)) == want_d


def _chains(ka, a):
    return [a] if ka == "linestring" else a


@pytest.mark.parametrize("ka", ["linestring", "multilinestring"])
@pytest.mark.parametrize("kb", ["polygon", "multipolygon"])
def test_length_partition_is_exact(ka, kb):
    A, B = pf.family_a(ka, kb, 24)
    for a, b in zip(A, B):
        whole = sum((abs(F(q[0]) - F(p[0])) + abs(F(q[1]) - F(p[1])) for ch in _chains(ka, a) for p, q in zip(ch, ch[1:])), F(0))
        assert cr.l1(cr.clip(ka, a, kb, b)) + cr.l1(cr.clip(ka, a, kb, b, invert=True)) == whole
        eu = sum(math.dist(p, q) for ch in _chains(ka, a) for p, q in zip(ch, ch[1:]))
        assert math.isclose(cr.length(ka, a, kb, b) + cr.length(ka, a, kb, b, invert=True), eu, rel_tol=1e-12, abs_tol=1e-12)


@pytest.mark.parametrize("ka", ["point", "multipoint"])
@pytest.mark.parametrize("kb", ["polygon", "multipolygon"])
def test_point_partition(ka, kb):
    A, B = pf.family_a(ka, kb, 24)
    for a, b in zip(A, B):
        pts = [a] if ka == "point" else list(a)
        inside, outside = cr.clip(ka, a, kb, b), cr.clip(ka, a, kb, b, invert=True)
        assert sorted(inside + outside) == sorted(pts)
        assert inside == [p for p in pts if p in inside] and outside == [p for p in pts if p in outside]  # input order
