"""The CPU reference of the nearest join (tests/nearest_reference.py): its brute-force arm and its ring-search arm agree
bit for bit on every right type, with null / empty / NaN / unbounded rows planted, lattice ties, points outside the box,
non-finite and null points, max_distance limits and degenerate boxes."""
import math

import numpy as np
import pytest

import nearest_reference as nr
import shapes
from geopolars_b200 import GeoArrowArray, GeometryType
from test_gpu_nearest import T, planted, query_points


def both_arms(a, P, pvalid=None, maxd=math.inf):
    b = nr.nearest_join(a, P, pvalid, maxd, use_grid=False)
    g = nr.nearest_join(a, P, pvalid, maxd, use_grid=True)
    assert np.array_equal(b[0], g[0])
    assert np.array_equal(b[1].view(np.int64), g[1].view(np.int64))
    assert np.array_equal(b[2], g[2])
    return b


@pytest.mark.parametrize("kind", list(T))
def test_arms_agree_on_every_type(conv, kind):
    rng = np.random.default_rng(100 + list(T).index(kind))
    rows = shapes.random_rows(rng, kind, 120) + planted(kind, rng)
    rows = [rows[i] for i in rng.permutation(len(rows))]
    a = conv(GeoArrowArray.from_shapes(T[kind], rows))
    P = query_points(rng, 60)
    pvalid = np.ones(len(P), bool)
    pvalid[::11] = False
    nid, dist, tied = both_arms(a, P, pvalid)
    assert (nid[~pvalid] == -1).all() and (nid[-3:] == -1).all()  # null and non-finite points
    far = np.arange(len(P) - 10, len(P) - 7)
    assert (nid[far[pvalid[far]]] >= 0).all()  # points far outside the box
    both_arms(a, P, pvalid, maxd=1.0)
    both_arms(a, P, pvalid, maxd=0.0)


def test_lattice_ties_and_degenerate_boxes(conv):
    g = np.arange(12, dtype=np.float64)
    X, Y = np.meshgrid(g, g)
    lat = conv(GeoArrowArray.points(np.stack([X.ravel(), Y.ravel()], 1)))
    P = np.stack(np.meshgrid(np.arange(11) + 0.5, np.arange(11) + 0.5), -1).reshape(-1, 2)
    _, dist, tied = both_arms(lat, P)
    assert (tied == 4).all() and (dist == math.hypot(0.5, 0.5)).all()
    rng = np.random.default_rng(7)
    xs = np.sort(rng.uniform(0, 100, 80))
    flat = conv(GeoArrowArray.from_shapes(GeometryType.LINESTRING, [[(x, 0.0), (x + 0.5, 0.0)] for x in xs]))
    both_arms(flat, np.concatenate([rng.uniform(-10, 110, (40, 2)), [[50.0, 0.0], [1e6, 0.0]]]))
    same = conv(GeoArrowArray.points(np.full((20, 2), 1.25)))
    nid, _, tied = both_arms(same, rng.uniform(-5, 5, (10, 2)))
    assert (tied == 20).all() and (nid == 0).all()
    one = conv(GeoArrowArray.from_shapes(GeometryType.POLYGON, [shapes.random_polygon(rng)]))
    both_arms(one, rng.uniform(-20, 30, (20, 2)))


def test_reference_rejects_invalid_max_distance(conv):
    a = conv(GeoArrowArray.points(np.zeros((2, 2))))
    for bad in (math.nan, -1.0):
        with pytest.raises(ValueError):
            nr.nearest_join(a, np.zeros((1, 2)), max_distance=bad)
