"""Symmetric difference, the remainders and the five overlay modes (DESIGN.md §4.23) on the GPU: ring for ring agreement with
the exact referees (overlay_modes_reference.py), bit for bit agreement of one-cutter and no-cutter remainders with the
row-wise difference, the area identities, partitions and the union's total area on the bundled datasets and the stars, the
row order, OGC validity of every row, nulls, errors and determinism, and GeoDataFrame.overlay."""
import numpy as np
import pytest

import boolean_reference as br
import overlay_modes_reference as omr
import pairs_families as pf
import validity_reference as vr
from geopolars_b200 import GeoArrowArray, GeometryType, _lib, datasets, engine, synth
from geopolars_b200.geoseries import GeoDataFrame, GeoSeries, overlay
from test_gpu_boolean import check_form, grid_cells, row_areas, rows, same_rings
from test_gpu_dissolve import local_areas
from test_gpu_overlay import gather
from test_overlay_area_model import case_pairs

P, MP = GeometryType.POLYGON, GeometryType.MULTIPOLYGON
HOWS = ("intersection", "union", "identity", "symmetric_difference", "difference")
ABSENT = np.uint64(0xFFFFFFFFFFFFFFFF)


def upload(ctx, t, rws):
    return ctx.upload(GeoArrowArray.from_shapes(t, rws))


def fl(members):
    return [[[tuple(map(float, p)) for p in r] for r in m] for m in members]


def canon(members):
    """members ordered by their shell's first two vertices: members whose shells start at one point (pieces of A - B and
    B - A meeting at a vertex) are in the kernel's tracing order there, which the output form leaves open"""
    return sorted(members, key=lambda m: [(float(x), float(y)) for x, y in m[0][:2]])


def valid_rows(d):
    reason, valid = engine.is_valid(d)
    return bool(valid.all() and (reason == 0).all())


def host_bytes(d):
    h = d.to_host()
    return (np.asarray(h.xy).tobytes(), np.asarray(h.geom_off).tobytes(), np.asarray(h.part_off).tobytes(), np.asarray(h.ring_off).tobytes())


def stars(shift=(0.0, 0.0)):
    xy, ro, go = synth.star_polygons()
    return GeoArrowArray.polygons(xy + np.array(shift), ro, go)


# ---- symmetric difference ------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_symmetric_difference_hand_cases_exact(ctx):
    cases = omr.symmetric_difference_hand_cases()
    da, db = upload(ctx, MP, [c[0] for c in cases]), upload(ctx, MP, [c[1] for c in cases])
    d = engine.boolean_op(da, db, "symmetric_difference")
    assert valid_rows(d)
    for (a, b, want), got in zip(cases, rows(d)):
        check_form(got)
        assert got == fl(want), (a, b, got)
    assert rows(engine.boolean_op(db, da, "symmetric_difference")) == rows(d)


def _check_symdiff(ctx, pairs):
    A, B = [a for a, _ in pairs], [b for _, b in pairs]
    d = engine.boolean_op(upload(ctx, MP, A), upload(ctx, MP, B), "symmetric_difference")
    assert valid_rows(d)
    for i, got in enumerate(rows(d)):
        check_form(got)
        want = omr.symmetric_difference(A[i], B[i])
        assert same_rings(canon(got), canon(want), A[i], B[i]), (i, A[i], B[i], got, br.as_float(want))
    return d


@pytest.mark.gpu
def test_symmetric_difference_referee_on_model_pairs_and_column_types(ctx):
    pairs = case_pairs()[:400]
    d = _check_symdiff(ctx, pairs)
    # Polygon and MultiPolygon columns give the same bytes
    single = [i for i, (a, b) in enumerate(pairs) if len(a) == 1 and len(b) == 1]
    want = host_bytes(ctx.upload(gather(d.to_host(), single)))
    pa, pb = upload(ctx, P, [pairs[i][0][0] for i in single]), upload(ctx, P, [pairs[i][1][0] for i in single])
    ma, mb = upload(ctx, MP, [pairs[i][0] for i in single]), upload(ctx, MP, [pairs[i][1] for i in single])
    for x, y in ((pa, pb), (pa, mb), (ma, pb), (ma, mb)):
        assert host_bytes(engine.boolean_op(x, y, "symmetric_difference")) == want


@pytest.mark.gpu
@pytest.mark.parametrize("offset", range(len(pf.A_OFFSETS)))
def test_symmetric_difference_referee_on_lattice_pairs(ctx, offset):
    ox, oy = pf.A_OFFSETS[offset]
    ra, rb = pf.family_a("polygon", "multipolygon", 40)
    _check_symdiff(ctx, [([pf.translate(a, ox, oy)], pf.translate(b, ox, oy)) for a, b in zip(ra, rb)])


@pytest.mark.gpu
def test_symmetric_difference_area_identity_on_the_stars(ctx):
    a, b = ctx.upload(stars()), ctx.upload(stars((3.0, 2.0)))
    d = engine.boolean_op(a, b, "symmetric_difference")
    assert valid_rows(d)
    ia, ok = engine.intersection_area(a, b)
    aa, ab = np.abs(local_areas(a)), np.abs(local_areas(b))  # ring by ring from its first vertex: no cancellation
    got = local_areas(d)
    assert ok.all() and np.all(np.abs(got - (aa + ab - 2 * ia)) <= 1e-12 * (aa + ab))


@pytest.mark.gpu
def test_symmetric_difference_nulls_row_independence_and_determinism(ctx):
    sq = br._sq
    A = [[sq(0, 0, 2)], None, [], [sq(0, 0, 2)], [[(0, 0), (np.nan, 0), (1, 1), (0, 0)]], [sq(0, 0, 2)], []]
    B = [[sq(1, 1, 2)], [sq(0, 0, 1)], [sq(0, 0, 1)], None, [sq(0, 0, 1)], [], []]
    got = rows(engine.boolean_op(upload(ctx, P, A), upload(ctx, P, B), "symmetric_difference"))
    assert [r is None for r in got] == [False, True, False, True, True, False, False]
    assert got[2] == [[sq(0.0, 0.0, 1.0)]] and got[5] == [[sq(0.0, 0.0, 2.0)]] and got[6] == []
    s = GeoSeries(_device=upload(ctx, P, A)).geo.symmetric_difference(GeoSeries(_device=upload(ctx, P, B)))
    assert isinstance(s, GeoSeries) and rows(s.device) == got
    pairs = case_pairs()[:200]
    A, B = [a for a, _ in pairs], [b for _, b in pairs]
    full = rows(engine.boolean_op(upload(ctx, MP, A), upload(ctx, MP, B), "symmetric_difference"))
    again = rows(engine.boolean_op(upload(ctx, MP, A), upload(ctx, MP, B), "symmetric_difference"))
    part = rows(engine.boolean_op(upload(ctx, MP, A[50:60]), upload(ctx, MP, B[50:60]), "symmetric_difference"))
    assert full == again and full[50:60] == part
    with pytest.raises(ValueError):
        engine.boolean_op(upload(ctx, MP, A), upload(ctx, MP, B), "xor")


# ---- remainders ----------------------------------------------------------------------------------------------------------

def _left_remainders(ctx, lhs, rhs):
    """{i: row} of overlay(lhs, rhs, "difference")"""
    a, b, g = engine.overlay(lhs, rhs, "difference")
    assert np.all(b == ABSENT) and np.all(np.diff(a.astype(np.int64)) > 0)
    return dict(zip(a.astype(np.int64).tolist(), rows(g))), g


@pytest.mark.gpu
def test_remainder_with_one_cutter_is_the_rowwise_difference(ctx):
    a, b = stars(), stars((3.0, 2.0))
    li, ri, _ = engine.overlay_join(ctx.upload(a), ctx.upload(b))
    # distinct subjects and cutters, then only the rows whose one cutter is their partner
    _, first = np.unique(li, return_index=True)
    li, ri = li[first], ri[first]
    _, first = np.unique(ri, return_index=True)
    li, ri = li[first], ri[first]
    sa, sb = ctx.upload(gather(a, li.astype(np.int64))), ctx.upload(gather(b, ri.astype(np.int64)))
    pl, pr = engine.spatial_join(sa, sb, "intersects")
    cnt = np.bincount(pl.astype(np.int64), minlength=len(li))
    own = np.zeros(len(li), dtype=bool)
    own[pl[pl == pr].astype(np.int64)] = True
    keep = np.nonzero((cnt == 1) & own)[0]
    assert len(keep) > 1000
    sa, sb = ctx.upload(gather(sa.to_host(), keep)), ctx.upload(gather(sb.to_host(), keep))
    rem, g = _left_remainders(ctx, sa, sb)
    want = rows(engine.boolean_op(sa, sb, "difference"))
    assert len(rem) == sum(1 for w in want if w)
    for i, w in enumerate(want):
        assert rem.get(i, []) == w, i
    assert valid_rows(g)
    # no cutter: the difference with an empty row
    far = ctx.upload(stars((1e6, 0.0)))
    rem, _ = _left_remainders(ctx, sa, far)
    want = rows(engine.boolean_op(sa, upload(ctx, P, [[]] * len(keep)), "difference"))
    assert [rem[i] for i in range(len(keep))] == want


def _remainder_groups():
    """(subject, cutters) groups: the hand cases, then model rows with 2 to 6 cutters each"""
    groups = [(s, c) for s, c, _ in omr.remainder_hand_cases()]
    pairs = case_pairs(60)
    k, sizes = 0, (2, 3, 4, 5, 6)
    for t in range(40):
        m = sizes[t % len(sizes)]
        groups.append((pairs[k][0], [pairs[k + u][1] for u in range(m)]))
        k += m
    return groups


def _translate(members, dx):
    return [[[(x + dx, y) for x, y in r] for r in m] for m in members]


@pytest.mark.gpu
def test_remainder_groups_agree_with_the_fold(ctx):
    groups = _remainder_groups()
    subj, cut, owner = [], [], []
    for g, (s, cs) in enumerate(groups):  # groups far apart: each subject meets only its own cutters
        subj.append(_translate(s, 4096.0 * g))
        for c in cs:
            cut.append(_translate(c, 4096.0 * g))
            owner.append(g)
    # a null subject and a non-finite subject over group 0's cutters, a null and a non-finite cutter over subject 0
    subj += [None, [[[(0, 0), (np.nan, 0), (1, 1), (0, 0)]]]]
    cut += [None, [[[(0, 0), (4, 0), (np.inf, 4), (0, 0)]]]]
    rem, g = _left_remainders(ctx, upload(ctx, MP, subj), upload(ctx, MP, cut))
    assert valid_rows(g)
    assert len(groups) not in rem and len(groups) + 1 not in rem
    for k, (s, _) in enumerate(groups):
        cs = [c for c, o in zip(cut, owner) if o == k]
        want = omr.remainder(subj[k], cs)
        got = rem.get(k, [])
        check_form(got)
        assert vr.validity_code("multipolygon", got) == 0
        assert same_rings(canon(got), canon(want), subj[k], [m for c in cs for m in c]), (k, got, br.as_float(want))


# ---- overlay -------------------------------------------------------------------------------------------------------------

def _parts(ctx, lhs, rhs):
    """the three kinds of rows, each as {(lhs, rhs): row}, built from overlay_join and the difference mode of both orders"""
    li, ri, g = engine.overlay_join(lhs, rhs)
    inter = dict(zip(zip(li.tolist(), ri.tolist()), rows(g)))
    a, _, g = engine.overlay(lhs, rhs, "difference")
    left = {(i, int(ABSENT)): r for i, r in zip(a.tolist(), rows(g))}
    b, _, g = engine.overlay(rhs, lhs, "difference")
    right = {(int(ABSENT), j): r for j, r in zip(b.tolist(), rows(g))}
    return inter, left, right


@pytest.mark.gpu
def test_every_mode_is_the_union_of_its_parts_in_order(ctx):
    lhs, rhs = ctx.upload(stars()), ctx.upload(stars((3.0, 2.0)))
    inter, left, right = _parts(ctx, lhs, rhs)
    table = {"intersection": (inter,), "difference": (left,), "identity": (inter, left), "symmetric_difference": (left, right),
             "union": (inter, left, right)}
    for how in HOWS:
        a, b, g = engine.overlay(lhs, rhs, how)
        keys = list(zip(a.tolist(), b.tolist()))
        assert keys == sorted(keys) and len(set(keys)) == len(keys), how
        want = {}
        for part in table[how]:
            want.update(part)
        assert keys == sorted(want), how
        assert rows(g) == [want[k] for k in keys], how
        assert valid_rows(g), how
        a2, b2, g2 = engine.overlay(lhs, rhs, how)
        assert np.array_equal(a, a2) and np.array_equal(b, b2) and host_bytes(g) == host_bytes(g2), how
    a, b, g = engine.overlay(lhs, rhs, "intersection")
    li, ri, gj = engine.overlay_join(lhs, rhs)
    assert np.array_equal(a, li) and np.array_equal(b, ri) and host_bytes(g) == host_bytes(gj)


def _check_left_partition(ctx, left, right):
    """every left row: its intersection areas plus its remainder's area equal its area"""
    a, b, g = engine.overlay(left, right, "identity")
    assert valid_rows(g)
    sums = np.bincount(a.astype(np.int64), weights=row_areas(g), minlength=len(left))
    area = np.abs(engine.area(left))
    assert np.all(np.abs(sums - area) <= 1e-9 * area), np.max(np.abs(sums - area) / area)
    return len(a)


@pytest.mark.gpu
def test_identity_partitions_naturalearth_by_a_5_degree_grid(ctx):
    d = datasets.read_dataset("naturalearth_lowres").geometry.device
    reason, _ = engine.is_valid(d)
    keep = np.nonzero(reason == 0)[0]
    left = ctx.upload(gather(d.to_host(), keep))
    assert _check_left_partition(ctx, left, upload(ctx, P, grid_cells(-180.0, -90.0, 5.0, 72, 36))) > len(keep)


@pytest.mark.gpu
def test_identity_partitions_the_stars_by_a_200_grid(ctx):
    left = ctx.upload(stars())
    assert _check_left_partition(ctx, left, upload(ctx, P, grid_cells(0.0, 0.0, 5.0, 200, 200))) > 10_000


@pytest.mark.gpu
def test_union_total_area_is_the_union_of_both_columns(ctx):
    a, b = stars(), stars((3.0, 2.0))
    k = np.arange(300)
    a, b = gather(a, k), gather(b, k)
    lhs, rhs = ctx.upload(a), ctx.upload(b)
    _, _, g = engine.overlay(lhs, rhs, "union")
    assert valid_rows(g)
    both = ctx.upload(GeoArrowArray.from_shapes(MP, [r for r in rows(engine.boolean_op(lhs, upload(ctx, P, [[]] * 300), "union"))] +
                                                [r for r in rows(engine.boolean_op(rhs, upload(ctx, P, [[]] * 300), "union"))]))
    total = float(row_areas(engine.union_all(both))[0])
    assert abs(row_areas(g).sum() - total) <= 1e-9 * total


@pytest.mark.gpu
def test_overlay_errors_come_before_any_launch(ctx):
    lhs = upload(ctx, P, [[br._sq(0, 0, 1)]])
    pts = ctx.upload(GeoArrowArray.from_shapes(GeometryType.POINT, [(0, 0)]))
    n0 = ctx.launch_count
    with pytest.raises(ValueError):
        engine.overlay(lhs, lhs, "xor")
    with pytest.raises(_lib.MismatchedGeometry):
        engine.overlay(lhs, pts, "union")
    with pytest.raises(_lib.MismatchedGeometry):
        engine.overlay(pts, lhs, "difference")
    import ctypes as C

    hp, ha = C.c_void_p(), C.c_void_p()
    assert ctx.lib.gpl_overlay(ctx._h, lhs._h, lhs._h, 5, C.byref(hp), C.byref(ha)) == -7
    assert hp.value is None and ha.value is None
    assert ctx.launch_count == n0


@pytest.mark.gpu
def test_geoseries_and_geodataframe_overlay(ctx):
    import pyarrow as pa

    sq = br._sq
    L = [[sq(0, 0, 2)], [sq(10, 0, 1)]]
    R = [[sq(1, 1, 2)], [sq(20, 0, 1)]]
    ls, rs = GeoSeries(_device=upload(ctx, P, L)), GeoSeries(_device=upload(ctx, P, R))
    a, b, g = overlay(ls, rs, "union")
    assert a.dtype == np.int64 and b.dtype == np.int64 and isinstance(g, GeoSeries)
    assert a.tolist() == [0, 0, 1, -1, -1] and b.tolist() == [0, -1, -1, 0, 1]
    a2, b2, g2 = overlay(ls, rs, "intersection")
    assert a2.tolist() == [0] and b2.tolist() == [0]
    left = GeoDataFrame(pa.table({"name": ["a", "b"], "x": [1, 2], "geometry": ls.device.to_arrow()}))
    right = GeoDataFrame(pa.table({"name": ["p", "q"], "y": [10.0, 20.0], "geometry": rs.device.to_arrow()}))
    out = left.overlay(right, how="union")
    assert out.columns == ["name_1", "x", "name_2", "y", "geometry"] and len(out) == 5
    assert out["name_1"].to_pylist() == ["a", "a", "b", None, None]
    assert out["x"].to_pylist() == [1, 1, 2, None, None]
    assert out["name_2"].to_pylist() == ["p", None, None, "p", "q"]
    assert out["y"].to_pylist() == [10.0, None, None, 10.0, 20.0]
    assert rows(out.geometry.device) == rows(g.device)
    out = left.overlay(right, how="difference")
    assert out.columns == ["name_1", "x", "name_2", "y", "geometry"] and out["name_2"].to_pylist() == [None, None]
    # a right column named as the left geometry
    right = GeoDataFrame(pa.table({"geometry": ["p", "q"], "shape": rs.device.to_arrow()}), geometry="shape")
    out = left.overlay(right, how="intersection")
    assert out.columns == ["name", "x", "geometry_2", "geometry"] and out["geometry_2"].to_pylist() == ["p"]
