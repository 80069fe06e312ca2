"""The exact DE-9IM referee (tests/relate_reference.py) on hand-derived matrices, and its invariants on valid random pairs of
all 36 type pairs (tests/pairs_families.py family A): transposition, EE = 2, entries bounded by the parts' dimensions, within
/ contains / geom_equals consistency, and agreement with the exact oracle's intersects and contains (tests/pairs_reference.py)."""
import pytest

import pairs_families as PF
import pairs_reference as PR
import relate_reference as R


def sq(x, y, s):
    return [(x, y), (x + s, y), (x + s, y + s), (x, y + s), (x, y)]


HAND = [
    ("polygon", [sq(0, 0, 1)], "polygon", [[(1, 0), (2, 0), (2, 1), (1, 1), (1, 0)]], "FF2F11212"),  # shared edge
    ("polygon", [sq(0, 0, 1)], "polygon", [sq(1, 1, 1)], "FF2F01212"),  # shared corner
    ("polygon", [sq(0, 0, 1)], "polygon", [[(1, 0), (0, 0), (0, 1), (1, 1), (1, 0)]], "2FFF1FFF2"),  # moved start, reversed
    ("polygon", [sq(0, 0, 4)], "polygon", [sq(1, 1, 1)], "212FF1FF2"),
    ("polygon", [sq(0, 0, 2)], "polygon", [sq(1, 1, 2)], "212101212"),
    ("linestring", [(-1, 0.5), (2, 0.5)], "polygon", [sq(0, 0, 1)], "101FF0212"),
    ("point", (0.5, 0.5), "polygon", [sq(0, 0, 1)], "0FFFFF212"),
    ("linestring", [(0, 0), (2, 2)], "linestring", [(0, 2), (2, 0)], "0F1FF0102"),
    ("linestring", sq(0, 0, 1), "point", (0.5, 0), "0F1FFFFF2"),  # a closed ring has no boundary
    ("multilinestring", [[(0, 0), (1, 0)], [(1, 0), (2, 0)]], "point", (1, 0), "0F1FF0FF2"),  # Mod-2 rule
    ("polygon", [], "polygon", [sq(0, 0, 1)], "FFFFFF212"),  # empty
]


@pytest.mark.parametrize("ka,a,kb,b,want", HAND)
def test_hand_cases(ka, a, kb, b, want):
    assert R.relate(ka, a, kb, b) == want
    assert R.relate(kb, b, ka, a) == R.transpose(want)


def _part_dims(kind):
    d = R.dims(kind)
    return [d, d - 1 if d > 0 else -1, 2]  # interior, boundary (a point has none), exterior


@pytest.mark.parametrize("ka", PF.KINDS)
def test_invariants_on_random_pairs(ka):
    n = 28  # 6 x 6 type pairs x 28 rows ~ 1000 pairs over the six parametrizations
    for kb in PF.KINDS:
        ra, rb = PF.family_a(ka, kb, n)
        da, db = R.dims(ka), R.dims(kb)
        for a, b in zip(ra, rb):
            m = R.relate(ka, a, kb, b)
            mt = R.relate(kb, b, ka, a)
            assert mt == R.transpose(m), (ka, a, kb, b)
            assert m[8] == "2"
            pa, pb = _part_dims(ka), _part_dims(kb)
            for r in range(3):
                for c in range(3):
                    v = m[3 * r + c]
                    if v != "F":
                        assert int(v) <= min(pa[r], pb[c]), (ka, a, kb, b, m)
            within = R.predicate("within", m, da, db)
            contains_ba = R.predicate("contains", mt, db, da)
            assert within == contains_ba
            eq = R.predicate("geom_equals", m, da, db)
            assert eq == (da == db and within and R.predicate("contains", m, da, db))
            assert R.predicate("intersects", m, da, db) == PR.intersects(a, b, ka, kb), (ka, a, kb, b, m)
            if R.CLASS[ka] >= 1 and kb == "point":
                assert R.predicate("contains", m, da, db) == PR.contains_point(ka, a, b), (ka, a, kb, b, m)
            if R.CLASS[ka] == 2 and kb == "polygon":
                assert R.predicate("contains", m, da, db) == PR.contains_polygon(ka, a, b), (ka, a, kb, b, m)
