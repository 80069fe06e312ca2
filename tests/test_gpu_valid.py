"""gpl_is_valid on the GPU: code for code against the exact referee (tests/validity_reference.py) on the known answers, random
lattice rows, the bundled datasets and large rows; conventions, type coverage, row independence, determinism, errors and the
GeoSeries accessors."""
import ctypes as C
import math
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from shapes import sq  # noqa: E402
from test_validity_reference_cpu import known_answers, lattice_rows  # noqa: E402
from validity_reference import MESSAGES, validity_code  # noqa: E402

pytestmark = pytest.mark.gpu

from geopolars_b200 import GeoArrowArray, GeometryType, synth  # noqa: E402
from geopolars_b200 import engine as E  # noqa: E402

KIND = {"point": GeometryType.POINT, "multipoint": GeometryType.MULTIPOINT, "linestring": GeometryType.LINESTRING,
        "multilinestring": GeometryType.MULTILINESTRING, "polygon": GeometryType.POLYGON, "multipolygon": GeometryType.MULTIPOLYGON}


@pytest.fixture(scope="module")
def ctx():
    return E.Context(0)


def gpu_codes(ctx, kind, rows):
    reason, valid = E.is_valid(ctx.upload(GeoArrowArray.from_shapes(KIND[kind], rows)))
    return [int(c) if v else None for c, v in zip(reason, valid)]


def as_multi(row):
    return None if row is None else [row]


def test_known_answers(ctx):
    for kind in KIND:
        cases = [(row, want) for k, row, want in known_answers() if k == kind]
        if cases:
            assert gpu_codes(ctx, kind, [r for r, _ in cases]) == [w for _, w in cases], kind
    polys = [(row, want) for k, row, want in known_answers() if k == "polygon"]
    assert gpu_codes(ctx, "multipolygon", [as_multi(r) for r, _ in polys]) == [w for _, w in polys]


def test_random_lattice_rows_match_the_referee(ctx):
    rows = lattice_rows(np.random.default_rng(18), 2400)
    want_p = [(r, validity_code(k, r)) for k, r in rows if k == "polygon"]
    want_m = [(r, validity_code(k, r)) for k, r in rows if k == "multipolygon"]
    assert gpu_codes(ctx, "polygon", [r for r, _ in want_p]) == [w for _, w in want_p]
    assert gpu_codes(ctx, "multipolygon", [r for r, _ in want_m]) == [w for _, w in want_m]
    # the Polygon rows again as one-member MultiPolygons
    assert gpu_codes(ctx, "multipolygon", [[r] for r, _ in want_p]) == [w for _, w in want_p]


def test_unclosed_rings_give_the_codes_of_closed_rings(ctx):
    rows = [r for k, r in lattice_rows(np.random.default_rng(5), 600) if k == "polygon"]
    opened = [[ring[:-1] if len(ring) > 1 and tuple(ring[0]) == tuple(ring[-1]) else ring for ring in r] for r in rows]
    assert gpu_codes(ctx, "polygon", rows) == gpu_codes(ctx, "polygon", opened)


def polygon_shapes(a):
    """rows of a host Polygon / MultiPolygon GeoArrowArray in from_shapes nesting (MultiPolygon rows as lists of polygons)"""
    xy, ro = a.xy, a.ring_off

    def poly(r0, r1):
        return [[tuple(p) for p in xy[ro[g]:ro[g + 1]].tolist()] for g in range(r0, r1)]

    if a.type == GeometryType.POLYGON:
        return [poly(a.geom_off[i], a.geom_off[i + 1]) for i in range(len(a.geom_off) - 1)]
    po = a.part_off
    return [[poly(po[m], po[m + 1]) for m in range(a.geom_off[i], a.geom_off[i + 1])] for i in range(len(a.geom_off) - 1)]


@pytest.mark.parametrize("name", ["nybb", "naturalearth_lowres"])
def test_bundled_datasets_match_the_referee(ctx, name):
    from geopolars_b200 import datasets

    d = datasets.read_dataset(name).geometry.device
    host = d.to_host()
    kind = {GeometryType.POLYGON: "polygon", GeometryType.MULTIPOLYGON: "multipolygon"}[GeometryType(int(host.type))]
    reason, valid = E.is_valid(d)
    want = [validity_code(kind, r) for r in polygon_shapes(host)]
    assert valid.all() and reason.tolist() == want


def test_stars_and_blobs_are_valid_and_planted_defects_are_found(ctx):
    xy, ro, go = synth.star_polygons(10_000, 100)
    arr = GeoArrowArray.polygons(xy, ro, go)
    reason, valid = E.is_valid(ctx.upload(arr))
    assert valid.all() and (reason == 0).all()
    bxy, bro, bgo = synth.blob_polygons(1_000_000, nvert=32)
    reason, _ = E.is_valid(ctx.upload(GeoArrowArray.polygons(bxy, bro, bgo)))
    assert (reason == 0).all()
    # a defect in every 7th star: swap two consecutive vertices (a bow-tie, unless the radii let it stay simple) or add a spike
    xy2 = xy.copy()
    rows = np.arange(0, len(go) - 1, 7)
    for i, r in enumerate(rows):
        c0 = ro[go[r]]
        if i % 2 == 0:
            xy2[[c0 + 2, c0 + 3]] = xy2[[c0 + 3, c0 + 2]]
        else:
            xy2[c0 + 2] = xy2[c0 + 4]
    arr2 = GeoArrowArray.polygons(xy2, ro, go)
    reason, _ = E.is_valid(ctx.upload(arr2))
    want = np.zeros(len(reason), np.int8)
    for r in rows:
        want[r] = validity_code("polygon", [[tuple(p) for p in xy2[ro[go[r]]:ro[go[r] + 1]].tolist()]])
    assert (want[rows[1::2]] == 5).all() and (want[rows[::2]] == 5).any()
    assert np.array_equal(reason, want)


def test_large_rows(ctx):
    n = 1_000_000
    t = 2 * np.pi * np.arange(n) / n
    ring = np.stack([np.cos(t) * 1000.0, np.sin(t) * 1000.0], 1)
    assert gpu_codes(ctx, "polygon", [[ring.tolist()]]) == [0]
    bad = ring.copy()
    bad[[1000, 1001]] = bad[[1001, 1000]]  # two consecutive vertices swapped: their neighbouring edges cross
    assert gpu_codes(ctx, "polygon", [[bad.tolist()]]) == [5]
    holes = [sq(3 * i + 1, 3 * j + 1, 1) for i in range(100) for j in range(100)]
    shell = sq(0, 0, 301)
    assert gpu_codes(ctx, "polygon", [[shell] + holes]) == [0]
    touching = [(0, 0.5), (0.5, 0), (0.5, 0.5), (0, 0.5)]  # touches the shell twice, in the corner left free by the grid
    assert gpu_codes(ctx, "polygon", [[shell] + holes + [touching]]) == [4]


def test_every_type_nulls_and_empties(ctx):
    assert gpu_codes(ctx, "point", [(1, 2), None, (math.nan, math.nan), (math.inf, 0)]) == [0, None, 0, 10]
    assert gpu_codes(ctx, "multipoint", [[(1, 2)], None, [], [(math.nan, math.nan)]]) == [0, None, 0, 10]
    assert gpu_codes(ctx, "linestring", [[(0, 0), (1, 1)], None, [], [(1, 1), (1, 1)], [(0, 0)]]) == [0, None, 0, 9, 9]
    assert gpu_codes(ctx, "multilinestring", [[[(0, 0), (1, 1)]], None, [], [[(0, 0), (1, 1)], [(2, 2), (2, 2)]]]) == [0, None, 0, 9]
    assert gpu_codes(ctx, "polygon", [[sq(0, 0, 1)], None, [], [[]], [[], sq(0, 0, 1)]]) == [0, None, 0, 0, 2]
    assert gpu_codes(ctx, "multipolygon", [[[sq(0, 0, 1)]], None, [], [[]], [[], [sq(0, 0, 1)]]]) == [0, None, 0, 0, 0]
    assert gpu_codes(ctx, "polygon", []) == []


def test_row_independence_and_determinism(ctx):
    rows = [r for k, r in lattice_rows(np.random.default_rng(9), 1200) if k == "multipolygon"]
    arr = GeoArrowArray.from_shapes(GeometryType.MULTIPOLYGON, rows)
    d = ctx.upload(arr)
    full, _ = E.is_valid(d)
    again, _ = E.is_valid(d)
    assert full.tobytes() == again.tobytes()
    part = gpu_codes(ctx, "multipolygon", rows[37:311])
    assert part == full[37:311].tolist()


def test_invalid_arguments(ctx):
    lib = ctx.lib
    d = ctx.upload(GeoArrowArray.from_shapes(GeometryType.POLYGON, [[sq(0, 0, 1)]]))
    buf = np.zeros(1, np.int8)
    p = buf.ctypes.data_as(C.c_void_p)
    launches = ctx.launch_count
    assert lib.gpl_is_valid(None, d._h, p, None, 0) == -7
    assert lib.gpl_is_valid(ctx._h, None, p, None, 0) == -7
    assert lib.gpl_is_valid(ctx._h, d._h, None, None, 0) == -7
    assert ctx.launch_count == launches


def test_accessors(ctx):
    import pyarrow as pa

    from geopolars_b200.geoseries import GeoSeries

    rows = [[sq(0, 0, 1)], None, [[(0, 0), (2, 2), (2, 0), (0, 2), (0, 0)]], [sq(0, 0, 4), sq(5, 5, 1)]]
    s = GeoSeries(_device=ctx.upload(GeoArrowArray.from_shapes(GeometryType.POLYGON, rows)))
    v = s.geo.is_valid()
    assert v.type == pa.bool_() and v.to_pylist() == [True, None, False, False]
    r = s.geo.is_valid_reason()
    assert r.type == pa.string() and r.to_pylist() == [MESSAGES[0], None, MESSAGES[5], MESSAGES[2]]
