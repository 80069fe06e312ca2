"""Intersection, union and difference geometry and the geometry overlay join (DESIGN.md §4.19) on the GPU: ring for ring
agreement with the exact-rational referee (boolean_reference.py) on its hand cases and on the 900+ model pairs in all four
column-type combinations, area identities on the bundled datasets, OGC validity of every output row by the §4.18 kernel,
partitions at scale, shared edges and vertices at scale, nulls / empties / errors, invalid operands, row independence and
the join against the row-wise op."""
import numpy as np
import pytest

import boolean_reference as br
import overlay_reference as ref
import shapes
from geopolars_b200 import GeoArrowArray, GeometryType, _lib, datasets, engine, synth
from geopolars_b200.geoseries import GeoSeries, overlay_join
from test_gpu_overlay import gather
from test_overlay_area_model import case_pairs, known_cases

P, MP = GeometryType.POLYGON, GeometryType.MULTIPOLYGON
OPS = ("intersection", "union", "difference")
sq = shapes.sq


def upload(ctx, t, rows):
    return ctx.upload(GeoArrowArray.from_shapes(t, rows))


def rows(d):
    """a MultiPolygon DeviceArray -> per row None or [[ring, ...], ...] with rings as lists of (x, y)"""
    h = d.to_host()
    assert h.type == MP
    valid = np.ones(len(h), dtype=bool) if h.validity_bitmap() is None else np.unpackbits(h.validity_bitmap(), bitorder="little")[: len(h)].astype(bool)
    xy = np.asarray(h.xy, dtype=np.float64).reshape(-1, 2)
    out = []
    for i in range(len(h)):
        if not valid[i]:
            out.append(None)
            continue
        members = []
        for m in range(h.geom_off[i], h.geom_off[i + 1]):
            members.append([[tuple(map(float, p)) for p in xy[h.ring_off[r]:h.ring_off[r + 1]]] for r in range(h.part_off[m], h.part_off[m + 1])])
        out.append(members)
    return out


def shoelace(ring):
    return 0.5 * sum(a[0] * b[1] - b[0] * a[1] for a, b in zip(ring[:-1], ring[1:]))


def row_area(members):
    return sum(shoelace(m[0]) + sum(shoelace(h) for h in m[1:]) for m in members)


def tol(a, b):
    pts = np.array([p for m in (a, b) for rings in m for r in rings for p in r], dtype=np.float64).reshape(-1, 2)
    diag = float(np.hypot(*(pts.max(0) - pts.min(0)))) if len(pts) else 0.0
    return 1e-9 * float(ref.polygon_area(a) + ref.polygon_area(b)) + 1e-12 * diag * diag


def check_form(members):
    """closed rings, shells counter-clockwise and holes clockwise, each starting at its smallest vertex, no repeated
    consecutive coordinate, holes ordered by first vertex and members by their shell's first vertex"""
    firsts = []
    for m in members:
        for k, r in enumerate(m):
            assert len(r) >= 4 and r[0] == r[-1], r
            assert r[0] == min(r), r
            assert all(p != q for p, q in zip(r[:-1], r[1:])), r
            assert (shoelace(r) > 0) == (k == 0), r
        assert [h[0] for h in m[1:]] == sorted(h[0] for h in m[1:])
        firsts.append(m[0][0])
    assert firsts == sorted(firsts)


def all_valid(ctx, d):
    reason, valid = engine.is_valid(d)
    return reason


def same_rings(got, want, a, b):
    """got (GPU, floats) has want's (referee, Fractions) members and rings with the same cyclic vertex sequence: input
    vertices bit for bit, constructed crossing points within 1e-12 L (L: the diagonal of the union of the two envelopes)"""
    inputs = {(float(x), float(y)) for m in (a, b) for rings in m for r in rings for x, y in r}
    pts = np.array(sorted(inputs), dtype=np.float64).reshape(-1, 2)
    tol_l = 1e-12 * float(np.hypot(*(pts.max(0) - pts.min(0)))) if len(pts) else 0.0

    def close(g, w):
        wf = (float(w[0]), float(w[1]))
        if wf in inputs and w[0] == br.F(wf[0]) and w[1] == br.F(wf[1]):
            return g == wf
        return abs(g[0] - wf[0]) <= tol_l and abs(g[1] - wf[1]) <= tol_l

    if got is None or len(got) != len(want):
        return False
    for gm, wm in zip(got, want):
        if len(gm) != len(wm):
            return False
        for gr, wr in zip(gm, wm):
            if len(gr) != len(wr):
                return False
            g, w = gr[:-1], wr[:-1]
            if not any(all(close(g[(k + i) % len(g)], w[i]) for i in range(len(w))) for k in range(len(g))):
                return False
    return True


@pytest.mark.gpu
def test_hand_cases_exact_rings(ctx):
    cases = br.hand_cases()
    A = [c[0] for c in cases]
    B = [c[1] for c in cases]
    res = {op: rows(engine.boolean_op(upload(ctx, MP, A), upload(ctx, MP, B), op)) for op in OPS}
    for i, (a, b, op, want) in enumerate(cases):
        got = res[op][i]
        check_form(got)
        assert got == [[[tuple(map(float, p)) for p in r] for r in m] for m in want], (i, got)
    for op in OPS:
        reason = all_valid(ctx, engine.boolean_op(upload(ctx, MP, A), upload(ctx, MP, B), op))
        assert (reason == 0).all(), (op, reason)


def _pairs():
    return case_pairs() + [(a, b) for a, b, _ in known_cases() if a and b]


@pytest.mark.gpu
@pytest.mark.parametrize("op", OPS)
def test_referee_agreement_validity_and_type_combinations(ctx, op):
    pairs = _pairs()
    A, B = [a for a, _ in pairs], [b for _, b in pairs]
    da, db = upload(ctx, MP, A), upload(ctx, MP, B)
    d = engine.boolean_op(da, db, op)
    got = rows(d)
    reason, valid = engine.is_valid(d)
    assert valid.all() and (reason == 0).all(), (op, [(i, pairs[i]) for i in np.nonzero(reason)[0][:3]])
    for i, (a, b) in enumerate(pairs):
        want = br.boolean_op(a, b, op)
        check_form(got[i])
        assert same_rings(got[i], want, a, b), (op, i, a, b, got[i], br.as_float(want))
        assert abs(row_area(got[i]) - float(br.area(want))) <= tol(a, b), (op, i, row_area(got[i]), br.area(want))
    # the same rows from Polygon and MultiPolygon columns in all four combinations: the same bytes
    single = [i for i, (a, b) in enumerate(pairs) if len(a) == 1 and len(b) == 1]
    pa = upload(ctx, P, [pairs[i][0][0] for i in single])
    pb = upload(ctx, P, [pairs[i][1][0] for i in single])
    ma = upload(ctx, MP, [pairs[i][0] for i in single])
    mb = upload(ctx, MP, [pairs[i][1] for i in single])
    ref_rows = [got[i] for i in single]
    for x, y in ((pa, pb), (pa, mb), (ma, pb), (ma, mb)):
        assert rows(engine.boolean_op(x, y, op)) == ref_rows


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["nybb", "naturalearth_lowres"])
def test_datasets_against_intersection_area(ctx, name):
    d = datasets.read_dataset(name).geometry.device
    reason, _ = engine.is_valid(d)
    host = d.to_host()
    keep = np.nonzero(reason == 0)[0]
    a = ctx.upload(gather(host, keep))
    b = ctx.upload(gather(host, np.roll(keep, -1)))
    inter, _ = engine.intersection_area(a, b)
    aa, ab = np.abs(engine.area(a)), np.abs(engine.area(b))
    want = {"intersection": inter, "union": aa + ab - inter, "difference": aa - inter}
    for op in OPS:
        out = engine.boolean_op(a, b, op)
        r, _ = engine.is_valid(out)
        assert (r == 0).all(), (op, np.nonzero(r)[0])
        got = np.array([row_area(m) for m in rows(out)])
        scale = aa + ab
        assert np.all(np.abs(got - want[op]) <= 1e-9 * scale), (op, np.max(np.abs(got - want[op]) / scale))


@pytest.mark.gpu
def test_nulls_empties_nonfinite_and_errors(ctx):
    A = [[sq(0, 0, 2)], None, [], [sq(0, 0, 2)], [[(0, 0), (np.nan, 0), (1, 1), (0, 0)]], [sq(0, 0, 2)], [], [sq(0, 0, 2)]]
    B = [[sq(1, 1, 2)], [sq(0, 0, 1)], [sq(0, 0, 1)], None, [sq(0, 0, 1)], [], [], [[(0, 0), (1, 0), (np.inf, 1), (0, 0)]]]
    da, db = upload(ctx, P, A), upload(ctx, P, B)
    got = {op: rows(engine.boolean_op(da, db, op)) for op in OPS}
    for op in OPS:
        assert [r is None for r in got[op]] == [False, True, False, True, True, False, False, True]
    assert got["intersection"][2] == [] and got["intersection"][5] == [] and got["intersection"][6] == []
    assert got["union"][2] == [[sq(0.0, 0.0, 1.0)]] and got["union"][5] == [[sq(0.0, 0.0, 2.0)]]
    assert got["difference"][2] == [] and got["difference"][5] == [[sq(0.0, 0.0, 2.0)]]
    s = GeoSeries(_device=da)
    for op in OPS:
        out = getattr(s.geo, op)(GeoSeries(_device=db))
        assert isinstance(out, GeoSeries) and out.device.type == MP
    pts = ctx.upload(GeoArrowArray.from_shapes(GeometryType.POINT, [(0, 0)] * len(A)))
    with pytest.raises(_lib.MismatchedGeometry, match=r"Expected \(Multi\)Polygon x \(Multi\)Polygon"):
        engine.boolean_op(da, pts, "union")
    with pytest.raises(_lib.MismatchedGeometry):
        engine.overlay_join(pts, da)
    with pytest.raises(_lib.ShapeError):
        engine.boolean_op(da, upload(ctx, P, B[:3]), "intersection")
    with pytest.raises(ValueError):
        engine.boolean_op(da, db, "xor")


@pytest.mark.gpu
def test_invalid_operands_are_well_formed(ctx):
    bow = [(0, 0), (2, 2), (2, 0), (0, 2), (0, 0)]
    spike = [(0, 0), (2, 0), (2, 2), (1, 2), (1, 3), (1, 2), (0, 2), (0, 0)]
    pinch = [(0, 0), (4, 0), (4, 4), (2, 0), (0, 4), (0, 0)]
    A = [[bow], [spike], [pinch], [sq(0, 0, 2), sq(1, 1, 2)]]
    B = [[sq(1, 1, 2)], [sq(0, 0, 2)], [sq(1, -1, 2)], [sq(0, 0, 1)]]
    for op in OPS:
        h = engine.boolean_op(upload(ctx, P, A), upload(ctx, P, B), op).to_host()
        assert np.all(np.diff(h.geom_off) >= 0) and np.all(np.diff(h.part_off) >= 0) and np.all(np.diff(h.ring_off) >= 4)
        xy = np.asarray(h.xy).reshape(-1, 2)
        for r in range(len(h.ring_off) - 1):
            assert tuple(xy[h.ring_off[r]]) == tuple(xy[h.ring_off[r + 1] - 1])


@pytest.mark.gpu
def test_row_independence_and_determinism(ctx):
    pairs = _pairs()[:200]
    A, B = [a for a, _ in pairs], [b for _, b in pairs]
    for op in OPS:
        full = rows(engine.boolean_op(upload(ctx, MP, A), upload(ctx, MP, B), op))
        again = rows(engine.boolean_op(upload(ctx, MP, A), upload(ctx, MP, B), op))
        part = rows(engine.boolean_op(upload(ctx, MP, A[50:60]), upload(ctx, MP, B[50:60]), op))
        assert full == again and full[50:60] == part


@pytest.mark.gpu
def test_overlay_join_against_rowwise_and_area_join(ctx):
    rng = np.random.default_rng(7)
    L = [[shapes.valid_star(rng, float(x), float(y), 3.0, 9)] for x, y in rng.uniform(0, 20, (60, 2))]
    R = [[sq(float(i), float(j), 2.0)] for i in range(0, 24, 2) for j in range(0, 24, 2)]
    dl, dr = upload(ctx, P, L), upload(ctx, P, R)
    li, ri, g = engine.overlay_join(dl, dr)
    assert np.all(np.diff(li.astype(np.int64) * len(R) + ri.astype(np.int64)) > 0)
    got = rows(g)
    assert all(len(m) > 0 for m in got)
    assert (engine.is_valid(g)[0] == 0).all()
    rw = rows(engine.boolean_op(ctx.upload(gather(dl.to_host(), li)), ctx.upload(gather(dr.to_host(), ri)), "intersection"))
    assert got == rw
    al, ar, area = engine.overlay_area_join(dl, dr)
    kept = set(zip(li.tolist(), ri.tolist()))
    for i, j, v in zip(al.tolist(), ar.tolist(), area.tolist()):
        if (i, j) not in kept:
            assert v <= 1e-9 * 50
    assert kept <= set(zip(al.tolist(), ar.tolist()))
    # partition: the pieces of each left row sum to its area
    sums = np.zeros(len(L))
    for i, m in zip(li.tolist(), got):
        sums[i] += row_area(m)
    area_l = np.abs(engine.area(dl))
    inside = np.array([all(0 <= x <= 24 and 0 <= y <= 24 for x, y in r[0]) for r in L])
    assert np.all(np.abs(sums - area_l)[inside] <= 1e-9 * area_l[inside])
    li2, ri2, g2 = engine.overlay_join(dl, dr)
    h1, h2 = g.to_host(), g2.to_host()
    assert np.array_equal(li, li2) and np.array_equal(ri, ri2) and np.array_equal(np.asarray(h1.xy), np.asarray(h2.xy))
    a, b, s = overlay_join(GeoSeries(_device=dl), GeoSeries(_device=dr))
    assert a.dtype == np.int64 and b.dtype == np.int64 and isinstance(s, GeoSeries)


def row_areas(d):
    """the shoelace area of every row of a MultiPolygon DeviceArray (holes negative), vectorised"""
    h = d.to_host()
    xy = np.asarray(h.xy, dtype=np.float64).reshape(-1, 2)
    ro, po, go = np.asarray(h.ring_off), np.asarray(h.part_off), np.asarray(h.geom_off)
    if len(xy) == 0:
        return np.zeros(len(go) - 1)
    term = xy[:-1, 0] * xy[1:, 1] - xy[1:, 0] * xy[:-1, 1]
    csum = np.concatenate([[0.0], np.cumsum(term)])
    ring = 0.5 * (csum[ro[1:] - 1] - csum[ro[:-1]])  # the terms inside each ring (its last coordinate closes it)
    rc = np.concatenate([[0.0], np.cumsum(ring)])
    member = rc[po[1:]] - rc[po[:-1]]
    mc = np.concatenate([[0.0], np.cumsum(member)])
    return mc[go[1:]] - mc[go[:-1]]


def grid_cells(x0, y0, w, nx, ny):
    return [[sq(x0 + i * w, y0 + j * w, w)] for j in range(ny) for i in range(nx)]


def check_partition(ctx, left, cells):
    """every output of overlay_join(left, cells) is valid and the output areas of each left row sum to its area"""
    li, ri, g = engine.overlay_join(left, ctx.upload(GeoArrowArray.from_shapes(P, cells)))
    reason, valid = engine.is_valid(g)
    assert valid.all() and (reason == 0).all(), np.nonzero(reason)[0][:5]
    sums = np.bincount(li.astype(np.int64), weights=row_areas(g), minlength=len(left))
    area = np.abs(engine.area(left))
    assert np.all(np.abs(sums - area) <= 1e-9 * area), np.max(np.abs(sums - area) / area)
    return len(li)


@pytest.mark.gpu
def test_partition_naturalearth_by_a_5_degree_grid(ctx):
    d = datasets.read_dataset("naturalearth_lowres").geometry.device
    reason, _ = engine.is_valid(d)
    keep = np.nonzero(reason == 0)[0]
    assert len(keep) > 150
    left = ctx.upload(gather(d.to_host(), keep))
    assert check_partition(ctx, left, grid_cells(-180.0, -90.0, 5.0, 72, 36)) > len(keep)


def stars():
    xy, ro, go = synth.star_polygons()
    return GeoArrowArray.polygons(xy, ro, go)


@pytest.mark.gpu
def test_partition_config2_stars_by_a_200_grid(ctx):
    left = ctx.upload(stars())
    reason, _ = engine.is_valid(left)
    assert (reason == 0).all()
    assert check_partition(ctx, left, grid_cells(0.0, 0.0, 5.0, 200, 200)) > 10_000


@pytest.mark.gpu
def test_config2_stars_shifted_by_one_grid_step(ctx):
    """the stars against the same stars shifted by one grid step (10.0 along x): star j shifted lands in the cell of star j + 1, whose vertices lie on the same rays from the same centre.  Then a family
    that shares edges and vertices outright: each star against itself with a contiguous half of its vertices pushed out
    radially (shared vertices at both ends of the kept half, shared edges along it)."""
    xy, ro, go = synth.star_polygons()
    a = ctx.upload(GeoArrowArray.polygons(xy, ro, go))
    shifted = xy + np.array([10.0, 0.0])
    b = ctx.upload(GeoArrowArray.polygons(shifted, ro, go))
    li, ri, g = engine.overlay_join(a, b)
    assert len(li) > 0 and (engine.is_valid(g)[0] == 0).all()
    la = np.abs(engine.area(a))
    inter, _ = engine.intersection_area(ctx.upload(gather(a.to_host(), li)), ctx.upload(gather(b.to_host(), ri)))
    assert np.all(np.abs(row_areas(g) - inter) <= 1e-9 * (la[li] + la[ri]))
    # shared edges and vertices: vertices 8..40 of every star pushed out by 1.5 about the cell centre
    m, nv = len(go) - 1, 64
    pts = xy.reshape(m, nv + 1, 2)
    j = np.arange(m)
    centre = np.stack([(j % 100 + 0.5) * 10.0, (j // 100 + 0.5) * 10.0], 1)[:, None, :]
    out = pts.copy()
    out[:, 8:41] = centre + 1.5 * (pts[:, 8:41] - centre)
    db = ctx.upload(GeoArrowArray.polygons(out.reshape(-1, 2), ro, go))
    assert (engine.is_valid(db)[0] == 0).all()
    inter, _ = engine.intersection_area(a, db)
    ab = np.abs(engine.area(db))
    want = {"intersection": inter, "union": la + ab - inter, "difference": la - inter}
    host_a, host_b = a.to_host(), db.to_host()
    for op in OPS:
        d = engine.boolean_op(a, db, op)
        assert (engine.is_valid(d)[0] == 0).all(), op
        assert np.all(np.abs(row_areas(d) - want[op]) <= 1e-9 * (la + ab)), op
        got = rows(d)
        for k in range(0, m, 500):  # a sample against the referee, ring for ring
            ra = [[[tuple(p) for p in np.asarray(host_a.xy).reshape(-1, 2)[ro[k]:ro[k + 1]].tolist()]]]
            rb = [[[tuple(p) for p in np.asarray(host_b.xy).reshape(-1, 2)[ro[k]:ro[k + 1]].tolist()]]]
            assert same_rings(got[k], br.boolean_op(ra, rb, op), ra, rb), (op, k)
