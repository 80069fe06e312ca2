"""Clipping of line and point columns by polygon columns, the intersection length and the clip / length joins
(DESIGN.md §4.22) on the GPU: the hand cases bit for bit in every column-type combination, member for member agreement with
the exact-rational referee (clip_reference.py) on valid lattice pairs, at ulp-scale gaps, far from the origin and at every
lane-grouping chain length, a referee-free cross-check against relate on random rows, the boundary identity and partitions on
the bundled datasets and config 3's walks, nulls / empties / errors, determinism and the joins against the row-wise ops."""
import math

import numpy as np
import pytest

import boolean_families as bf
import clip_reference as cr
import pairs_families as pf
import shapes
from geopolars_b200 import GeoArrowArray, GeometryType, _lib, datasets, engine, synth
from geopolars_b200.geoseries import GeoSeries, clip_join, overlay_length_join

T = GeometryType
KIND = {"point": T.POINT, "multipoint": T.MULTIPOINT, "linestring": T.LINESTRING, "multilinestring": T.MULTILINESTRING,
        "polygon": T.POLYGON, "multipolygon": T.MULTIPOLYGON}
LINES, AREAS = ("linestring", "multilinestring"), ("polygon", "multipolygon")


def upload(ctx, kind, rows):
    return ctx.upload(GeoArrowArray.from_shapes(KIND[kind], rows))


def _valid(h):
    bm = h.validity_bitmap()
    return np.ones(len(h), dtype=bool) if bm is None else np.unpackbits(bm, bitorder="little")[: len(h)].astype(bool)


def out_rows(d):
    """a MultiLineString / MultiPoint DeviceArray -> per row None or its members (lists of (x, y)) / points"""
    h = d.to_host()
    valid = _valid(h)
    xy = [tuple(map(float, p)) for p in np.asarray(h.xy, dtype=np.float64).reshape(-1, 2)]
    out = []
    for i in range(len(h)):
        if not valid[i]:
            out.append(None)
        elif h.type == T.MULTIPOINT:
            out.append(xy[h.geom_off[i]:h.geom_off[i + 1]])
        else:
            assert h.type == T.MULTILINESTRING
            out.append([xy[h.ring_off[m]:h.ring_off[m + 1]] for m in range(h.geom_off[i], h.geom_off[i + 1])])
    return out


def raw(d):
    h = d.to_host()
    return (np.asarray(h.geom_off).tolist(), None if h.ring_off is None else np.asarray(h.ring_off).tolist(),
            np.asarray(h.xy, dtype=np.float64).tobytes(), _valid(h).tolist())


def clip_both(ctx, ka, A, kb, B):
    a, b = upload(ctx, ka, A), upload(ctx, kb, B)
    return out_rows(engine.clip(a, b)), out_rows(engine.clip(a, b, invert=True))


# ---- hand cases and type combinations ----------------------------------------------------------------------------------
@pytest.mark.gpu
def test_hand_cases_bit_for_bit_in_every_type_combination(ctx):
    for single, multi in (("linestring", "multilinestring"), ("point", "multipoint")):
        cases = [c for c in cr.HAND if c[1] in (single, multi)]
        A = [c[2] if c[1] == multi else [c[2]] for c in cases]
        for kb in AREAS:
            B = [c[4] if kb == "polygon" else [c[4]] for c in cases]
            gi, gd = clip_both(ctx, multi, A, kb, B)
            for c, i_, d_ in zip(cases, gi, gd):
                assert i_ == c[5], (c[0], kb, i_)
                assert d_ == c[6], (c[0], kb, d_)
        # the cases of single rows: the same bytes from both left and both right column types
        one = [c for c in cases if c[1] == single]
        got = set()
        for ka in (single, multi):
            for kb in AREAS:
                a = upload(ctx, ka, [c[2] if ka == single else [c[2]] for c in one])
                b = upload(ctx, kb, [c[4] if kb == "polygon" else [c[4]] for c in one])
                got.add(repr((raw(engine.clip(a, b)), raw(engine.clip(a, b, invert=True)))))
        assert len(got) == 1


# ---- the referee --------------------------------------------------------------------------------------------------------
def check_against_referee(got_i, got_d, ka, A, kb, B, labels=None):
    bad = []
    for k, (a, b) in enumerate(zip(A, B)):
        for got, inv in ((got_i[k], False), (got_d[k], True)):
            msg = cr.matches(got, cr.clip(ka, a, kb, b, invert=inv))
            if msg:
                bad.append((labels[k] if labels else k, inv, msg))
    assert not bad, bad[:5]


@pytest.mark.gpu
@pytest.mark.parametrize("ka", LINES)
@pytest.mark.parametrize("kb", AREAS)
def test_family_a_against_the_referee(ctx, ka, kb):
    A, B = pf.family_a(ka, kb, 80)
    gi, gd = clip_both(ctx, ka, A, kb, B)
    check_against_referee(gi, gd, ka, A, kb, B)


@pytest.mark.gpu
def test_family_a_far_from_the_origin(ctx):
    for ka in LINES:
        for kb in AREAS:
            A, B = pf.family_a(ka, kb, 40)
            o_i, o_d = clip_both(ctx, ka, A, kb, B)
            for ox, oy in pf.A_OFFSETS[1:]:
                At, Bt = [pf.translate(a, ox, oy) for a in A], [pf.translate(b, ox, oy) for b in B]
                t_i, t_d = clip_both(ctx, ka, At, kb, Bt)
                for k in range(len(A)):
                    verts = set(_all_pts(At[k])) | set(_all_pts(Bt[k]))
                    for got, base in ((t_i[k], o_i[k]), (t_d[k], o_d[k])):
                        assert len(got) == len(base), (ka, kb, k, ox)
                        for m, m0 in zip(got, base):
                            assert len(m) == len(m0), (ka, kb, k, ox)
                            for p, p0 in zip(m, m0):
                                if p in verts:
                                    assert p == (p0[0] + ox, p0[1] + oy), (ka, kb, k, p, p0)
                                else:
                                    assert abs(p[0] - (p0[0] + ox)) <= math.ulp(p[0]) and abs(p[1] - (p0[1] + oy)) <= math.ulp(p[1]), (k, p, p0)


def _all_pts(row):
    if row is None:
        return []
    if isinstance(row, tuple):
        return [row]
    return [q for r in row for q in _all_pts(r)]


@pytest.mark.gpu
def test_family_b_ulp_gaps_against_the_referee(ctx):
    cases = [c for c in pf.family_b() if c[0] in LINES and c[2] in AREAS]
    assert len(cases) > 50
    for ka in LINES:
        for kb in AREAS:
            sel = [c for c in cases if c[0] == ka and c[2] == kb]
            A, B = [c[1] for c in sel], [c[3] for c in sel]
            gi, gd = clip_both(ctx, ka, A, kb, B)
            check_against_referee(gi, gd, ka, A, kb, B, labels=[(c[4], i) for i, c in enumerate(sel)])


@pytest.mark.gpu
def test_every_lane_grouping_length(ctx):
    o = bf.BC_OFFSET
    five = [(o + 1.0, o + 1.0), (o + 9.0, o + 2.0), (o + 10.0, o + 8.0), (o + 4.0, o + 11.0), (o + 0.5, o + 6.0), (o + 1.0, o + 1.0)]
    A, B = [], []
    for n in bf.BC_LENGTHS:
        # a zigzag of n edges across the pentagon, and the pentagon's edges as a line against an n-gon
        zig = [(o - 1.0 + 12.0 * i / n, o + (0.25 if i % 2 else 10.5) + 0.125 * (i % 3)) for i in range(n + 1)]
        ngon = [(o + 5.0 + 4.5 * math.cos(2 * math.pi * k / n), o + 5.0 + 4.5 * math.sin(2 * math.pi * k / n)) for k in range(n)]
        ngon = [(float(np.round(x * 64) / 64), float(np.round(y * 64) / 64)) for x, y in ngon]
        A += [zig, five]
        B += [[five], [ngon + [ngon[0]]]]
    gi, gd = clip_both(ctx, "linestring", A, "polygon", B)
    check_against_referee(gi, gd, "linestring", A, "polygon", B)


# ---- relate cross-check -------------------------------------------------------------------------------------------------
def collapsed(ka, a, kb, b, invert):
    """every member of the referee's clip rounds to fewer than 2 distinct points (rounding collapses the row's pieces)"""
    return all(len({(float(p[0]), float(p[1])) for p, _ in m}) < 2 for m in cr.clip(ka, a, kb, b, invert=invert))


def lattice_rows(rng, kind, n):
    """shapes' random rows on the exact dyadic lattice of pairs_families, so their touching and collinear relations hold"""
    return [pf._dyadic(r) for r in shapes.random_rows(rng, kind, n)]


@pytest.mark.gpu
def test_members_agree_with_relate_on_random_rows(ctx):
    """clip has a member iff relate's II or IB is '1', clip(invert) iff IE is '1', except where every piece of the
    referee's clip rounds to one point"""
    rng = np.random.default_rng(2204)
    for ka in LINES:
        for kb in AREAS:
            A, B = lattice_rows(rng, ka, 25_000), lattice_rows(rng, kb, 25_000)
            a, b = upload(ctx, ka, A), upload(ctx, kb, B)
            reason, _ = engine.is_valid(b)
            m, valid = engine.relate(a, b)
            gi, gd = out_rows(engine.clip(a, b)), out_rows(engine.clip(a, b, invert=True))
            rows = np.nonzero((reason == 0) & valid)[0]
            assert len(rows) > 5_000
            bad = []
            for k in rows:
                for got, want, inv in ((gi[k], m[k, 0] == 1 or m[k, 1] == 1, False), (gd[k], m[k, 2] == 1, True)):
                    if (len(got) > 0) != want and not (want and collapsed(ka, A[k], kb, B[k], inv)):
                        bad.append((ka, kb, int(k), inv, m[k].tolist()))
            assert not bad, bad[:5]


# ---- datasets -----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["nybb", "naturalearth_lowres"])
def test_boundary_identity_on_datasets(ctx, name):
    d = datasets.read_dataset(name).geometry.device
    reason, _ = engine.is_valid(d)
    h = d.to_host()
    xy = [tuple(map(float, p)) for p in np.asarray(h.xy, dtype=np.float64).reshape(-1, 2)]
    keep = np.nonzero(reason == 0)[0]
    assert len(keep) >= 5
    rings, polys = [], []
    for i in keep:
        if h.type == T.MULTIPOLYGON:
            members = [[xy[h.ring_off[r]:h.ring_off[r + 1]] for r in range(h.part_off[m], h.part_off[m + 1])] for m in range(h.geom_off[i], h.geom_off[i + 1])]
        else:
            members = [[xy[h.ring_off[r]:h.ring_off[r + 1]] for r in range(h.geom_off[i], h.geom_off[i + 1])]]
        rings.append(members[0][0])
        polys.append(members)
    a, b = upload(ctx, "linestring", rings), upload(ctx, "multipolygon", polys)
    gi, gd = out_rows(engine.clip(a, b)), out_rows(engine.clip(a, b, invert=True))
    for k, ring in enumerate(rings):
        assert gi[k] == [_dedup(ring)], (name, keep[k])
        assert gd[k] == [], (name, keep[k])


def _dedup(ring):
    return [p for i, p in enumerate(ring) if i == 0 or p != ring[i - 1]]


def grid_cells(x0, y0, w, nx, ny):
    return [[shapes.sq(x0 + i * w, y0 + j * w, w)] for j in range(ny) for i in range(nx)]


def check_length_partition(ctx, left, cells, mask=None):
    li, ri, length = engine.overlay_length_join(left, ctx.upload(GeoArrowArray.from_shapes(T.POLYGON, cells)))
    sums = np.bincount(li.astype(np.int64), weights=length, minlength=len(left))
    whole = engine.euclidean_length(left)
    sel = np.ones(len(left), dtype=bool) if mask is None else mask
    assert np.all(np.abs(sums - whole)[sel] <= 1e-9 * whole[sel]), np.max(np.abs(sums - whole)[sel] / np.maximum(whole[sel], 1e-300))
    return len(li)


@pytest.mark.gpu
def test_partition_naturalearth_exteriors_by_a_5_degree_grid(ctx):
    d = datasets.read_dataset("naturalearth_lowres").geometry.device
    reason, _ = engine.is_valid(d)
    h = d.to_host()
    xy = [tuple(map(float, p)) for p in np.asarray(h.xy, dtype=np.float64).reshape(-1, 2)]
    rings = []
    for i in np.nonzero(reason == 0)[0]:
        m = h.geom_off[i] if h.type == T.MULTIPOLYGON else None
        r = h.part_off[m] if m is not None else h.geom_off[i]
        rings.append(xy[h.ring_off[r]:h.ring_off[r + 1]])
    # a ring with an edge along an inner grid line is counted in the cells on both sides of it, and a ring reaching past
    # the antimeridian (x = 180 + 6e-14 in the data) is not covered by the grid
    on_line = lambda r: any((p[0] == q[0] and -180 < p[0] < 180 and p[0] % 5 == 0) or (p[1] == q[1] and -90 < p[1] < 90 and p[1] % 5 == 0)  # noqa: E731
                            for p, q in zip(r, r[1:]))
    covered = lambda r: all(-180 <= p[0] <= 180 and -90 <= p[1] <= 90 for p in r)  # noqa: E731
    mask = np.array([covered(r) and not on_line(r) for r in rings])
    assert mask.sum() > 0.9 * len(rings)
    left = upload(ctx, "linestring", rings)
    assert check_length_partition(ctx, left, grid_cells(-180.0, -90.0, 5.0, 72, 36), mask) > len(rings)


@pytest.mark.gpu
def test_partition_config3_walks_by_a_200_grid(ctx):
    xy, go = synth.walk_linestrings(20_000)
    left = ctx.upload(GeoArrowArray(T.LINESTRING, xy, geom_off=go))
    w = xy.reshape(-1, 16, 2)
    inside = (w.min(axis=(1, 2)) >= 0.0) & (w.max(axis=(1, 2)) < 1000.0)
    assert check_length_partition(ctx, left, grid_cells(0.0, 0.0, 5.0, 200, 200), inside) > 20_000


# ---- consistency, errors, determinism -----------------------------------------------------------------------------------
@pytest.mark.gpu
def test_clip_length_against_the_clip_and_the_difference(ctx):
    rng = np.random.default_rng(7)
    A, B = shapes.random_rows(rng, "multilinestring", 5_000), shapes.random_rows(rng, "multipolygon", 5_000)
    a, b = upload(ctx, "multilinestring", A), upload(ctx, "multipolygon", B)
    reason, _ = engine.is_valid(b)
    ln, valid = engine.clip_length(a, b)
    li = engine.euclidean_length(engine.clip(a, b))
    ld = engine.euclidean_length(engine.clip(a, b, invert=True))
    whole = engine.euclidean_length(a)
    ok = valid & (reason == 0)
    assert ok.sum() > 1_000
    assert np.all(ln[valid] >= 0.0)
    assert np.all(np.abs(ln - li)[ok] <= 1e-12 * whole[ok] + 1e-300)
    assert np.all(np.abs(li + ld - whole)[ok] <= 1e-12 * whole[ok] + 1e-300)


@pytest.mark.gpu
def test_nulls_empties_nonfinite_and_errors(ctx):
    sq = cr.SQ
    nan = float("nan")
    A = [None, [(-2.0, 2.0), (6.0, 2.0)], [], [(-2.0, 2.0), (6.0, 2.0)], [(nan, 2.0), (6.0, 2.0)], [(-2.0, 2.0), (6.0, 2.0)], [(1.0, 1.0)]]
    B = [[sq], None, [sq], [], [sq], [[(0.0, 0.0), (4.0, 0.0), (float("inf"), 4.0), (0.0, 0.0)]], [sq]]
    a, b = upload(ctx, "linestring", A), upload(ctx, "polygon", B)
    gi, gd = out_rows(engine.clip(a, b)), out_rows(engine.clip(a, b, invert=True))
    assert gi == [None, None, [], [], None, None, []]
    assert gd == [None, None, [], [[(-2.0, 2.0), (6.0, 2.0)]], None, None, []]
    ln, valid = engine.clip_length(a, b)
    assert valid.tolist() == [False, False, True, True, False, False, True]
    assert ln[2] == 0.0 and ln[3] == 0.0 and ln[6] == 0.0 and np.isnan(ln[~valid]).all()
    P = [[(1.0, 1.0), (5.0, 5.0)], None, [(nan, 0.0)], [], [(0.0, 0.0)]]
    p = upload(ctx, "multipoint", P)
    q = upload(ctx, "polygon", [[sq]] * 5)
    assert out_rows(engine.clip(p, q)) == [[(1.0, 1.0)], None, None, [], [(0.0, 0.0)]]
    assert out_rows(engine.clip(p, q, invert=True)) == [[(5.0, 5.0)], None, None, [], []]
    with pytest.raises(_lib.MismatchedGeometry):
        engine.clip(b, b)
    with pytest.raises(_lib.MismatchedGeometry):
        engine.clip(a, a)
    with pytest.raises(_lib.MismatchedGeometry):
        engine.clip_length(p, q)
    with pytest.raises(_lib.MismatchedGeometry):
        engine.overlay_length_join(p, q)
    with pytest.raises(_lib.ShapeError):
        engine.clip(a, upload(ctx, "polygon", [[sq]]))
    with pytest.raises(_lib.ShapeError):
        engine.clip_length(a, upload(ctx, "polygon", [[sq]]))
    # the polygon ops keep refusing line operands
    with pytest.raises(_lib.MismatchedGeometry):
        engine.boolean_op(a, b, "intersection")


@pytest.mark.gpu
def test_row_independence_and_determinism(ctx):
    rng = np.random.default_rng(11)
    A, B = shapes.random_rows(rng, "multilinestring", 3_000), shapes.random_rows(rng, "multipolygon", 3_000)
    a, b = upload(ctx, "multilinestring", A), upload(ctx, "multipolygon", B)
    for inv in (False, True):
        first = raw(engine.clip(a, b, invert=inv))
        assert raw(engine.clip(a, b, invert=inv)) == first
        whole = out_rows(engine.clip(a, b, invert=inv))
        part = out_rows(engine.clip(upload(ctx, "multilinestring", A[1000:1500]), upload(ctx, "multipolygon", B[1000:1500]), invert=inv))
        assert whole[1000:1500] == part
    l1, _ = engine.clip_length(a, b)
    l2, _ = engine.clip_length(a, b)
    assert l1.tobytes() == l2.tobytes()


# ---- joins --------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_joins_against_the_rowwise_ops(ctx):
    rng = np.random.default_rng(5)
    A = lattice_rows(rng, "multilinestring", 600)
    B = lattice_rows(rng, "polygon", 1200)
    a, b = upload(ctx, "multilinestring", A), upload(ctx, "polygon", B)
    reason, _ = engine.is_valid(b)
    B = [B[k] for k in np.nonzero(reason == 0)[0]]
    b = upload(ctx, "polygon", B)
    pi, pj = engine.predicate_join(a, b, "intersects")
    assert len(pi) > 200
    ga = upload(ctx, "multilinestring", [A[i] for i in pi])
    gb = upload(ctx, "polygon", [B[j] for j in pj])
    # overlay_length_join: the intersects pairs, each with the row-wise length bit for bit
    li, lj, lv = engine.overlay_length_join(a, b)
    assert np.array_equal(li, pi) and np.array_equal(lj, pj)
    want, valid = engine.clip_length(ga, gb)
    assert valid.all() and lv.tobytes() == want.tobytes()
    si, sj, sv = overlay_length_join(GeoSeries(_device=a), GeoSeries(_device=b), how="left")
    unmatched = np.setdiff1d(np.arange(len(A)), pi)
    assert len(si) == len(pi) + len(unmatched) and np.isnan(sv[sj == -1]).all() and np.array_equal(np.sort(si[sj == -1]), unmatched)
    # clip_join: the intersects pairs with a member (relate II or IB is 1), each with the row-wise clip bit for bit
    rowwise = out_rows(engine.clip(ga, gb))
    has = np.array([len(r) > 0 for r in rowwise])
    m, _ = engine.relate(ga, gb)
    rel = (m[:, 0] == 1) | (m[:, 1] == 1)
    assert all(collapsed("multilinestring", A[pi[k]], "polygon", B[pj[k]], False) for k in np.nonzero(has != rel)[0])
    ci, cj, cg = engine.clip_join(a, b)
    assert np.array_equal(ci, pi[has]) and np.array_equal(cj, pj[has])
    assert out_rows(cg) == [r for r, h in zip(rowwise, has) if h]
    ki, kj, ks = clip_join(GeoSeries(_device=a), GeoSeries(_device=b))
    assert np.array_equal(ki, ci.astype(np.int64)) and len(ks) == len(ci)
    # points: the pairs where some point lies in the closed polygon; for Point rows exactly covered_by
    P = lattice_rows(rng, "point", 2_000)
    p = upload(ctx, "point", P)
    qi, qj, qg = engine.clip_join(p, b)
    ci2, cj2 = engine.predicate_join(p, b, "covered_by")
    assert np.array_equal(qi, ci2) and np.array_equal(qj, cj2)
    assert out_rows(qg) == [[P[i]] for i in qi]


@pytest.mark.gpu
def test_geoseries_accessors(ctx):
    a = GeoSeries(_device=upload(ctx, "linestring", [[(-2.0, 2.0), (6.0, 2.0)], None]))
    b = GeoSeries(_device=upload(ctx, "polygon", [[cr.SQ], [cr.SQ]]))
    assert out_rows(a.geo.clip(b).device) == [[[(0.0, 2.0), (4.0, 2.0)]], None]
    assert out_rows(a.geo.clip(b, invert=True).device) == [[[(-2.0, 2.0), (0.0, 2.0)], [(4.0, 2.0), (6.0, 2.0)]], None]
    assert a.geo.intersection_length(b).to_pylist() == [4.0, None]
