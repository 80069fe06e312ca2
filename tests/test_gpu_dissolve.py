"""dissolve and union_all (DESIGN.md §4.21) on the GPU: two- and one-row groups bit for bit against the row-wise union, ring
for ring agreement with the exact referee (dissolve_reference.py) on model and hand groups, the overlay round trip (cut a
star by a grid, glue the pieces back), whole-column unions against inclusion-exclusion, and the semantics: nulls, skipped
rows, non-finite rows, empty groups, keys, errors, invalid rows, determinism and row order."""
import numpy as np
import pytest

import boolean_reference as br
import dissolve_reference as dr
import pairs_families as pf
import validity_reference as vr
from geopolars_b200 import GeoArrowArray, GeometryType, _lib, datasets, engine, synth
from geopolars_b200.geoseries import GeoDataFrame, GeoSeries, dissolve
from test_gpu_boolean import check_form, row_areas, rows, same_rings
from test_gpu_overlay import gather
from test_overlay_area_model import case_pairs

P, MP = GeometryType.POLYGON, GeometryType.MULTIPOLYGON


def upload(ctx, t, rws):
    return ctx.upload(GeoArrowArray.from_shapes(t, rws))


def star_columns(ctx, shift=(3.0, 2.0)):
    xy, ro, go = synth.star_polygons()
    return xy, ro, go, ctx.upload(GeoArrowArray.polygons(xy, ro, go)), ctx.upload(GeoArrowArray.polygons(xy + np.array(shift), ro, go))


def same_bytes(d1, d2):
    h1, h2 = d1.to_host(), d2.to_host()
    return (len(h1) == len(h2) and np.array_equal(np.asarray(h1.xy), np.asarray(h2.xy)) and np.array_equal(h1.geom_off, h2.geom_off)
            and np.array_equal(h1.part_off, h2.part_off) and np.array_equal(h1.ring_off, h2.ring_off)
            and (h1.valid is None) == (h2.valid is None) and (h1.valid is None or np.array_equal(h1.valid, h2.valid)))


@pytest.mark.gpu
def test_two_and_one_row_groups_are_the_rowwise_union(ctx):
    xy, ro, go, a, b = star_columns(ctx)
    n = len(go) - 1
    both = ctx.upload(GeoArrowArray.polygons(np.concatenate([xy, xy + np.array([3.0, 2.0])]), np.concatenate([ro, ro[1:] + ro[-1]]),
                                             np.arange(2 * n + 1, dtype=np.int64)))
    codes = np.concatenate([np.arange(n), np.arange(n)])
    got = engine.dissolve(both, codes, n)
    assert same_bytes(got, engine.boolean_op(a, b, "union"))
    # the lower row's edge first in every crossing: the same bytes with the shifted stars as the lower rows
    both_r = ctx.upload(gather(both.to_host(), np.concatenate([np.arange(n, 2 * n), np.arange(n)])))
    assert same_bytes(engine.dissolve(both_r, codes, n), engine.boolean_op(b, a, "union"))
    empty = upload(ctx, P, [[]] * n)
    assert same_bytes(engine.dissolve(a, np.arange(n), n), engine.boolean_op(a, empty, "union"))


def _groups(rws, sizes=(2, 3, 4, 5, 6)):
    out, k, s = [], 0, 0
    while k < len(rws):
        m = sizes[s % len(sizes)]
        out.append(rws[k:k + m])
        k, s = k + m, s + 1
    return out


def _check_groups(ctx, groups, exact=False):
    flat = [r for g in groups for r in g]
    codes = np.repeat(np.arange(len(groups)), [len(g) for g in groups])
    d = engine.dissolve(upload(ctx, MP, flat), codes, len(groups))
    reason, valid = engine.is_valid(d)
    assert valid.all() and (reason == 0).all(), [(i, groups[i]) for i in np.nonzero(reason)[0][:2]]
    got = rows(d)
    for i, g in enumerate(groups):
        want = dr.union_all(g)
        check_form(got[i])
        assert vr.validity_code("multipolygon", got[i]) == 0, (i, g, got[i])
        if exact:
            assert got[i] == br.as_float(want), (i, g, got[i], br.as_float(want))
        else:
            members = [m for r in g for m in r]
            assert same_rings(got[i], want, members, []), (i, g, got[i], br.as_float(want))
    return got


@pytest.mark.gpu
def test_referee_agreement_on_model_groups(ctx):
    pairs = case_pairs(60)
    rws = [r for a, b in pairs[:160] for r in (a, b)]
    _check_groups(ctx, _groups(rws))


@pytest.mark.gpu
@pytest.mark.parametrize("offset", range(len(pf.A_OFFSETS)))
def test_referee_agreement_on_lattice_groups(ctx, offset):
    ox, oy = pf.A_OFFSETS[offset]
    ra, rb = pf.family_a("polygon", "multipolygon", 40)
    rws = [m for a, b in zip(ra, rb) for m in ([pf.translate(a, ox, oy)], pf.translate(b, ox, oy))]
    _check_groups(ctx, _groups(rws, (2, 3, 4)))


@pytest.mark.gpu
def test_hand_groups_exact(ctx):
    groups = [g for g, _ in dr.hand_groups()]
    got = _check_groups(ctx, groups, exact=True)
    for (g, want), m in zip(dr.hand_groups(), got):
        if want is not None:
            assert m == [[[tuple(map(float, p)) for p in r] for r in mm] for mm in want]


def _grid(x0, y0, w, nx, ny):
    i, j = np.meshgrid(np.arange(nx, dtype=np.float64), np.arange(ny, dtype=np.float64), indexing="xy")
    xs, ys = x0 + i.ravel() * w, y0 + j.ravel() * w
    xy = np.stack([np.stack([xs, xs + w, xs + w, xs, xs], 1), np.stack([ys, ys, ys + w, ys + w, ys], 1)], 2).reshape(-1, 2)
    k = nx * ny
    return GeoArrowArray.polygons(xy, np.arange(k + 1, dtype=np.int64) * 5, np.arange(k + 1, dtype=np.int64))


def local_areas(d):
    """the shoelace area of every row of a (Multi)Polygon DeviceArray, each ring summed relative to its first vertex (no
    cancellation against the rest of the column)"""
    h = d.to_host()
    xy = np.asarray(h.xy, dtype=np.float64).reshape(-1, 2)
    ro = np.asarray(h.ring_off)
    po = np.asarray(h.part_off) if h.part_off is not None else np.arange(len(ro))
    go = np.asarray(h.geom_off)
    ring = np.zeros(len(ro) - 1)
    for k in range(len(ro) - 1):
        p = xy[ro[k]:ro[k + 1]] - xy[ro[k]]
        ring[k] = 0.5 * np.sum(p[:-1, 0] * p[1:, 1] - p[1:, 0] * p[:-1, 1])
    member = np.array([ring[po[m]:po[m + 1]].sum() for m in range(len(po) - 1)])
    return np.array([member[go[i]:go[i + 1]].sum() for i in range(len(go) - 1)])


def boundary_distance(out, left):
    """per row: the largest distance of a vertex of out (MultiPolygon) from the boundary of the same row of left, and the
    row's envelope diagonal"""
    ho, hl = out.to_host(), left.to_host()
    xo, xl = np.asarray(ho.xy).reshape(-1, 2), np.asarray(hl.xy).reshape(-1, 2)
    rl, gl = np.asarray(hl.ring_off), np.asarray(hl.geom_off)
    pl = np.asarray(hl.part_off) if hl.part_off is not None else np.arange(len(rl))
    ro, po, go = np.asarray(ho.ring_off), np.asarray(ho.part_off), np.asarray(ho.geom_off)
    worst, diag = np.zeros(len(gl) - 1), np.zeros(len(gl) - 1)
    for i in range(len(gl) - 1):
        r0, r1 = pl[gl[i]], pl[gl[i + 1]]
        segs = np.concatenate([np.stack([xl[rl[r]:rl[r + 1] - 1], xl[rl[r] + 1:rl[r + 1]]], 1) for r in range(r0, r1)])
        c0, c1 = ro[po[go[i]]], ro[po[go[i + 1]]]
        pts = xo[c0:c1]
        if len(pts) == 0:
            continue
        a, b = segs[None, :, 0], segs[None, :, 1]
        ab, ap = b - a, pts[:, None, :] - a
        t = np.clip(np.sum(ap * ab, 2) / np.maximum(np.sum(ab * ab, 2), 1e-300), 0.0, 1.0)
        d = np.hypot(*np.moveaxis(ap - t[..., None] * ab, 2, 0))
        worst[i] = d.min(1).max()
        lo, hi = segs.reshape(-1, 2).min(0), segs.reshape(-1, 2).max(0)
        diag[i] = np.hypot(*(hi - lo))
    return worst, diag


def _round_trip(ctx, left, cells):
    li, _, pieces = engine.overlay_join(left, ctx.upload(cells))
    back = engine.dissolve(pieces, li.astype(np.int64), len(left))
    reason, valid = engine.is_valid(back)
    assert valid.all() and (reason == 0).all(), np.nonzero(reason)[0][:5]
    area = np.abs(engine.area(left))
    return back, area, np.abs(row_areas(back))


@pytest.mark.gpu
def test_overlay_round_trip_on_a_dyadic_grid(ctx):
    xy, ro, go, stars, _ = star_columns(ctx)
    back, _, _ = _round_trip(ctx, stars, _grid(0.0, 0.0, 8.0, 128, 128))
    area, got = np.abs(local_areas(stars)), np.abs(local_areas(back))
    assert np.all(np.abs(got - area) <= 1e-12 * area), np.max(np.abs(got - area) / area)
    h = back.to_host()
    assert np.array_equal(np.diff(h.geom_off), np.ones(len(h), dtype=np.int64))  # one member per star
    assert np.array_equal(np.diff(h.part_off), np.ones(len(h), dtype=np.int64))  # no holes
    out = np.asarray(h.xy).reshape(-1, 2)
    for k in range(0, len(go) - 1, 97):  # every star vertex, bit for bit, on the star's ring
        ring = {tuple(p) for p in out[h.ring_off[k]:h.ring_off[k + 1]].tolist()}
        assert {tuple(p) for p in xy[ro[k]:ro[k + 1]].tolist()} <= ring, k


@pytest.mark.gpu
def test_overlay_round_trip_on_rounded_grids(ctx):
    _, _, _, stars, _ = star_columns(ctx)
    back, area, got = _round_trip(ctx, stars, _grid(0.0, 0.0, 5.0, 200, 200))
    assert np.all(np.abs(got - area) <= 1e-9 * area)
    worst, diag = boundary_distance(back, stars)  # no vertex off the star's boundary: no surviving sliver
    assert np.all(worst <= 1e-12 * diag), np.max(worst / diag)
    d = datasets.read_dataset("naturalearth_lowres").geometry.device
    reason, _ = engine.is_valid(d)
    left = ctx.upload(gather(d.to_host(), np.nonzero(reason == 0)[0]))
    back, area, got = _round_trip(ctx, left, _grid(-180.0, -90.0, 5.0, 72, 36))
    assert np.all(np.abs(got - area) <= 1e-9 * area), np.max(np.abs(got - area) / area)
    worst, diag = boundary_distance(back, left)
    assert np.all(worst <= 1e-12 * diag), np.max(worst / diag)


def _union_identity(ctx, col, check_triples):
    if check_triples:  # the identity below needs triple overlaps without area: each pairwise piece against every third row
        li, ri, pieces = engine.overlay_join(col, col)
        keep = np.nonzero(li < ri)[0]
        a, b, area3 = engine.overlay_area_join(ctx.upload(gather(pieces.to_host(), keep)), col)
        third = (b != li[keep][a]) & (b != ri[keep][a])
        assert area3[third].sum() <= 1e-10 * np.abs(engine.area(col)).sum(), area3[third].sum()
    u = engine.union_all(col)
    assert same_bytes(u, engine.dissolve(col, np.zeros(len(col), dtype=np.int64), 1))
    reason, valid = engine.is_valid(u)
    assert valid.all() and (reason == 0).all()
    li, ri, inter = engine.overlay_area_join(col, col)
    keep = li < ri
    area = np.abs(engine.area(col))
    want = area.sum() - inter[keep].sum()
    got = float(row_areas(u)[0])
    assert abs(got - want) <= 1e-9 * area.sum(), (got, want)
    return u


@pytest.mark.gpu
def test_union_all_of_naturalearth_and_of_the_stars(ctx):
    d = datasets.read_dataset("naturalearth_lowres").geometry.device
    reason, _ = engine.is_valid(d)
    _union_identity(ctx, ctx.upload(gather(d.to_host(), np.nonzero(reason == 0)[0])), True)
    # 300 stars and the same shifted by (3, 2): stars never overlap stars and shifted stars never overlap shifted stars, so
    # there are no triple overlaps.  (One group is assembled by one thread; DESIGN.md §4.21 has what 2 000 and 20 000 rows cost.)
    xy, ro, go = synth.star_polygons(m=300, grid=20)
    n = len(go) - 1
    both = ctx.upload(GeoArrowArray.polygons(np.concatenate([xy, xy + np.array([3.0, 2.0])]), np.concatenate([ro, ro[1:] + ro[-1]]),
                                             np.arange(2 * n + 1, dtype=np.int64)))
    _union_identity(ctx, both, False)


@pytest.mark.gpu
def test_nulls_skips_nonfinite_empties_keys_and_errors(ctx):
    sq = dr.sq
    A = [[sq(0, 0, 1)], None, [sq(1, 0, 1)], [sq(5, 5, 1)], [[(0, 0), (np.nan, 0), (1, 1), (0, 0)]], [sq(9, 9, 1)], [], None]
    codes = np.array([0, 0, 0, -1, 1, 1, 2, 3])
    got = rows(engine.dissolve(upload(ctx, P, A), codes, 5))
    assert got[0] == [[[(0.0, 0.0), (1.0, 0.0), (2.0, 0.0), (2.0, 1.0), (1.0, 1.0), (0.0, 1.0), (0.0, 0.0)]]]
    assert got[1] is None and got[2] == [] and got[3] == [] and got[4] == []
    assert rows(engine.union_all(upload(ctx, P, []))) == [[]]
    s = GeoSeries(_device=upload(ctx, P, A[:4]))
    u = s.geo.union_all()
    assert isinstance(u, GeoSeries) and len(u) == 1 and u.device.type == MP
    keys, g = dissolve(s, ["b", "a", None, "b"])
    assert keys.to_pylist() == ["a", "b"]
    assert rows(g.device) == [[], [[sq(0.0, 0.0, 1.0)], [sq(5.0, 5.0, 1.0)]]]
    keys, g = dissolve(s, np.array([7, 7, 3, 7]))
    assert keys.to_pylist() == [3, 7] and len(g) == 2
    import pyarrow as pa

    df = GeoDataFrame(pa.table({"k": [2, 1, 2, None], "geometry": s.device.to_arrow()}))
    out = df.dissolve("k")
    assert out.columns == ["k", "geometry"] and out["k"].to_pylist() == [1, 2] and len(out) == 2
    pts = ctx.upload(GeoArrowArray.from_shapes(GeometryType.POINT, [(0, 0)] * 3))
    n0 = ctx.launch_count
    with pytest.raises(_lib.MismatchedGeometry):
        engine.dissolve(pts, np.zeros(3, dtype=np.int64), 1)
    with pytest.raises(ValueError):
        engine.dissolve(s.device, np.zeros(3, dtype=np.int64), 1)
    with pytest.raises(ValueError):
        engine.dissolve(s.device, np.array([0, 1, 2, 3]), 3)
    with pytest.raises(ValueError):
        engine.dissolve(s.device, np.array([0, -2, 0, 0]), 3)
    assert ctx.launch_count == n0


@pytest.mark.gpu
def test_invalid_rows_are_well_formed(ctx):
    bow = [(0, 0), (2, 2), (2, 0), (0, 2), (0, 0)]
    spike = [(0, 0), (2, 0), (2, 2), (1, 2), (1, 3), (1, 2), (0, 2), (0, 0)]
    pinch = [(0, 0), (4, 0), (4, 4), (2, 0), (0, 4), (0, 0)]
    A = [[bow], [dr.sq(1, 1, 2)], [spike], [dr.sq(0, 0, 2)], [pinch], [dr.sq(1, -1, 2)], [dr.sq(0, 0, 2), dr.sq(1, 1, 2)]]
    h = engine.dissolve(upload(ctx, P, A), np.array([0, 0, 1, 1, 2, 2, 3]), 4).to_host()
    assert np.all(np.diff(h.geom_off) >= 0) and np.all(np.diff(h.part_off) >= 0) and np.all(np.diff(h.ring_off) >= 4)
    xy = np.asarray(h.xy).reshape(-1, 2)
    for r in range(len(h.ring_off) - 1):
        assert tuple(xy[h.ring_off[r]]) == tuple(xy[h.ring_off[r + 1] - 1])


@pytest.mark.gpu
def test_determinism_and_row_order(ctx):
    xy, ro, go, _, _ = star_columns(ctx)
    n = 2000
    both = ctx.upload(GeoArrowArray.polygons(np.concatenate([xy[:ro[n]], xy[:ro[n]] + np.array([3.0, 2.0])]),
                                             np.concatenate([ro[:n + 1], ro[1:n + 1] + ro[n]]), np.arange(2 * n + 1, dtype=np.int64)))
    codes = np.concatenate([np.arange(n) // 3, np.arange(n) // 3])
    ng = int(codes.max()) + 1
    first = engine.dissolve(both, codes, ng)
    assert same_bytes(first, engine.dissolve(both, codes, ng))
    perm = np.random.default_rng(5).permutation(2 * n)
    other = engine.dissolve(ctx.upload(gather(both.to_host(), perm)), codes[perm], ng)
    ga, gb = rows(first), rows(other)
    assert [[len(r) for r in m] for x in ga for m in x] == [[len(r) for r in m] for x in gb for m in x]
    for x, y in zip(ga, gb):
        for mx, my in zip(x, y):
            for rx, ry in zip(mx, my):
                assert np.max(np.abs(np.asarray(rx) - np.asarray(ry))) <= 1e-12 * 1000.0
