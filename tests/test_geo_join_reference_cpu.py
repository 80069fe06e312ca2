"""CPU checks of the great-circle joins' reference (tests/geo_join_reference.py): the vectorised oracle haversine against a
published value and the scalar entry point, and the cKDTree arms against their brute-force arms, bit for bit."""
import math

import numpy as np

import geo_join_reference as gref


def fixture(rng, n, m):
    """left and right lon/lat rows with an antimeridian cluster in both conventions, polar clusters, duplicates, lattice
    ties, nulls and out-of-range rows"""
    def cluster(c, k, s):
        return np.column_stack([c[0] + rng.uniform(-s, s, k), np.clip(c[1] + rng.uniform(-s, s, k), -90, 90)])

    Rr = np.concatenate([
        np.column_stack([rng.uniform(-180, 180, m), np.degrees(np.arcsin(rng.uniform(-1, 1, m)))]),
        cluster((179.9, 10.0), 30, 0.3), cluster((180.2, 10.0), 30, 0.3), cluster((0.0, 89.8), 20, 0.2), cluster((50.0, -89.9), 20, 0.1),
        [[10.0, 20.0], [10.0, 20.0], [12.0, 20.0], [8.0, 20.0], [0.0, 90.0], [77.0, 90.0]],
        [[np.nan, np.nan], [np.inf, 0.0], [0.0, 90.5], [360.5, 0.0], [5.0, np.nan]],
    ])
    L = np.concatenate([
        np.column_stack([rng.uniform(-180, 360, n), np.degrees(np.arcsin(rng.uniform(-1, 1, n)))]),
        [[180.0, 10.0], [-180.0, 10.0], [179.99, 10.1], [10.0, 20.0], [10.0, 25.0], [0.0, 90.0], [33.0, -90.0], [np.nan, np.nan], [0.0, -91.0]],
    ])
    lv, rv = np.ones(len(L), bool), np.ones(len(Rr), bool)
    lv[::11] = False
    rv[::13] = False
    return L, lv, Rr, rv


def test_vectorised_oracle_haversine(og):
    q = gref.haversine([[0.0, 0.0], [0.0, 0.0], [179.9, 0.0]], [[90.0, 0.0], [0.0, 90.0], [-179.9, 0.0]])
    assert abs(q[0] - 6371008.8 * math.pi / 2) < 1e-6 and abs(q[1] - 6371008.8 * math.pi / 2) < 1e-6  # a quarter great circle
    assert abs(q[2] - 0.2 * math.pi / 180 * 6371008.8) < 1e-6  # 0.2 degrees of the equator across the antimeridian (22 km)
    rng = np.random.default_rng(3)
    P = np.column_stack([rng.uniform(-360, 360, 200), rng.uniform(-90, 90, 200)])
    Q = np.column_stack([rng.uniform(-360, 360, 200), rng.uniform(-90, 90, 200)])
    d = gref.haversine(P, Q)
    want = np.array([og.geodesic_distance("haversine", *p, *q) for p, q in zip(P, Q)])
    assert np.array_equal(d.view(np.uint64), want.view(np.uint64))
    assert len(gref.haversine(np.zeros((0, 2)), np.zeros((0, 2)))) == 0


def test_tree_arms_agree_with_brute_force_bit_for_bit():
    L, lv, Rr, rv = fixture(np.random.default_rng(4), 60, 400)
    d_pair = gref.haversine([L[60 + 3]], [Rr[400 + 100 + 2]])[0]  # (10, 20) to (12, 20): D at a pair's distance
    for D in (0.0, 1.0, 3e4, d_pair, math.nextafter(d_pair, 0.0), 2e6, 1.5e7, math.pi * gref.R):
        a, b = gref.dwithin(L, Rr, D, lv, rv, tree=True), gref.dwithin(L, Rr, D, lv, rv, tree=False)
        for (ja, da), (jb, db) in zip(a, b):
            assert np.array_equal(ja, jb) and np.array_equal(da.view(np.uint64), db.view(np.uint64))
    i = 60 + 3
    assert 400 + 100 + 2 in gref.dwithin(L, Rr, d_pair, lv, rv)[i][0] and 400 + 100 + 2 not in gref.dwithin(L, Rr, math.nextafter(d_pair, 0.0), lv, rv)[i][0]
    for maxd in (math.inf, 0.0, 5e4, 3e6):
        na, da, ta = gref.nearest(L, Rr, maxd, lv, rv, tree=True)
        nb, db, tb = gref.nearest(L, Rr, maxd, lv, rv, tree=False)
        assert np.array_equal(na, nb) and np.array_equal(da.view(np.uint64), db.view(np.uint64))
        assert all(np.array_equal(x, y) for x, y in zip(ta, tb))
    nid, dist, ties = gref.nearest(L, Rr, math.inf, lv, rv)
    assert set(ties[60 + 3]) == {400 + 100, 400 + 100 + 1} and dist[60 + 3] == 0.0  # the duplicate rows at (10, 20)
    two = gref.dwithin(L, Rr, gref.haversine([[10.0, 20.0]], [[12.0, 20.0]])[0], lv, rv)[60 + 3]
    east, west = two[1][two[0] == 400 + 100 + 2], two[1][two[0] == 400 + 100 + 3]
    assert len(east) == 1 and east[0] == west[0]  # mirrored longitudes at one latitude: equal f64 distances
    assert nid[-1] == -1 and nid[-2] == -1 and np.all(nid[~gref.eligible(L, lv)] == -1)
    far = gref.nearest(L, Rr, 0.0, lv, rv)[0]
    assert far[60 + 3] == 400 + 100 and far[60 + 4] == -1


def test_out_of_range_null_and_empty_rows_never_match():
    L, lv, Rr, rv = fixture(np.random.default_rng(5), 20, 50)
    bad = np.nonzero(~gref.eligible(Rr, rv))[0]
    assert len(bad) >= 8
    for js, _ in gref.dwithin(L, Rr, math.pi * gref.R, lv, rv):
        assert not set(js) & set(bad)
    out = gref.dwithin(L, Rr, math.pi * gref.R, lv, rv)
    assert all(len(out[i][0]) == 0 for i in np.nonzero(~gref.eligible(L, lv))[0])
