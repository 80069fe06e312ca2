"""Intersection area (DESIGN.md §4.16) and the boolean geometry ops (§4.19) on the GPU over the families of
tests/boolean_families.py: far from the origin (BA), at ulp-scale gaps where constructed crossings round together (BB), at
every ring length where the lane grouping switches (BC) and on analytic answers at scale (BD).

  - intersection_area within the §4.16 tolerance of the exact referee, never negative, exactly 0.0 where the closures are
    disjoint, bit-identical under exact translation, and reproduced bit for bit by overlay_area_join;
  - every boolean output row valid by gpl_is_valid and by validity_reference; its exact (Fraction) shoelace area within
    perimeter · δ of the referee's exact area; every output vertex an input vertex bit for bit or within δ of a referee vertex,
    every referee vertex matched but those of a run the rounding collapsed (δ below);
  - BA: the same rings at every offset, input vertices bit for bit and constructed ones within 1 ulp of origin + offset;
  - BD bit for bit against the closed forms; unclosed BC rows give the bytes of closed ones; overlay_join against the
    row-wise op;
  - gpl_is_valid against validity_reference code for code on the referee's outputs rounded to doubles, invalid ones included.

δ of a crossing of input edges e and f: 2 ulp(max |c|) + 16 ε L |e||f| / |e × f| (ε = 2⁻⁵³, L the diagonal of the union of the
two rows' envelopes, max |c| over the row pair's coordinates): the rounding of the coordinates plus the error of t, which the
f64 orientations carry, magnified by the angle of the two edges."""
import math
from fractions import Fraction as F

import numpy as np
import pytest

import boolean_families as BF
import boolean_reference as br
import overlay_reference as ov
import pairs_reference as pr
import validity_reference as vr
from geopolars_b200 import GeoArrowArray, GeometryType, engine
from test_gpu_boolean import rows
from test_gpu_overlay import gather, tol

pytestmark = pytest.mark.gpu

T = {"polygon": GeometryType.POLYGON, "multipolygon": GeometryType.MULTIPOLYGON}
EPS = 2.0**-53
WORST = {"ratio": 0.0}


def by_types(ctx, cases, fn):
    """fn(col_a, col_b) -> per-row list, evaluated once per (kind_a, kind_b) group and scattered back into case order"""
    groups = {}
    for i, c in enumerate(cases):
        g = groups.setdefault((c[0], c[2]), ([], [], []))
        g[0].append(i), g[1].append(c[1]), g[2].append(c[3])
    out = [None] * len(cases)
    for (ka, kb), (idx, ra, rb) in groups.items():
        res = fn(ctx.upload(GeoArrowArray.from_shapes(T[ka], ra)), ctx.upload(GeoArrowArray.from_shapes(T[kb], rb)))
        for i, v in zip(idx, res):
            out[i] = v
    return out


def areas(ctx, cases):
    def fn(a, b):
        v, ok = engine.intersection_area(a, b)
        assert ok.all()
        return list(v)
    return np.array(by_types(ctx, cases, fn), dtype=np.float64)


def ops(ctx, cases, op):
    return by_types(ctx, cases, lambda a, b: rows(engine.boolean_op(a, b, op)))


def ops_codes(ctx, cases, op):
    def fn(a, b):
        d = engine.boolean_op(a, b, op)
        reason, valid = engine.is_valid(d)
        assert valid.all()
        return list(zip(rows(d), reason.tolist()))
    return by_types(ctx, cases, fn)


def mem(c):
    return BF.members(c[0], c[1]), BF.members(c[2], c[3])


def edges(m):
    return [(tuple(map(F, r[i])), tuple(map(F, r[(i + 1) % len(r)])))
            for p in m for ring in p for r in [vr.ring_vertices(ring)] for i in range(len(r))]


def _on(w, e):
    (px, py), (qx, qy) = e
    return ((qx - px) * (w[1] - py) - (qy - py) * (w[0] - px)) == 0 and min(px, qx) <= w[0] <= max(px, qx) and min(py, qy) <= w[1] <= max(py, qy)


def ulp(x):
    return math.ulp(abs(x)) if x else 5e-324


def row_scale(a, b):
    pts = np.array([p for m in (a, b) for poly in m for r in poly for p in r], dtype=np.float64).reshape(-1, 2)
    return float(np.abs(pts).max()), float(np.hypot(*(pts.max(0) - pts.min(0))))


def delta(w, ea, eb, cmax, L):
    """δ of the referee vertex w: 0 for an input vertex, else the bound of the crossing of the input edges it lies on"""
    worst = 0.0
    for e in ea:
        if not _on(w, e):
            continue
        for f in eb:
            if not _on(w, f):
                continue
            ex, ey = e[1][0] - e[0][0], e[1][1] - e[0][1]
            fx, fy = f[1][0] - f[0][0], f[1][1] - f[0][1]
            cr = abs(ex * fy - ey * fx)
            if cr == 0:
                continue
            le, lf = math.hypot(float(ex), float(ey)), math.hypot(float(fx), float(fy))
            worst = max(worst, 2 * ulp(cmax) + 16 * EPS * L * le * lf / float(cr))
    return worst


def exact_area(members):
    return sum((sum(F(p[0]) * F(q[1]) - F(q[0]) * F(p[1]) for p, q in zip(r[:-1], r[1:])) / 2 for m in members for r in m), F(0))


def perimeter(members):
    return sum(math.hypot(q[0] - p[0], q[1] - p[1]) for m in members for r in m for p, q in zip(r[:-1], r[1:]))


def check_geometry(c, got, want):
    """area and vertices of one output row against the referee's exact rings"""
    a, b = mem(c)
    cmax, L = row_scale(a, b)
    ea, eb = edges(a), edges(b)
    inputs = {(float(x), float(y)) for m in (a, b) for poly in m for r in poly for x, y in r}
    wv = list({p for m in want for r in m for p in r[:-1]})
    dl = [delta(w, ea, eb, cmax, L) for w in wv]
    for w, d in zip(wv, dl):
        if d == 0.0:
            assert (float(w[0]), float(w[1])) in inputs and F(float(w[0])) == w[0] and F(float(w[1])) == w[1], (c[4], w)
    gv = {p for m in got for r in m for p in r[:-1]}
    matched = set()
    for g in gv:
        if g in inputs:
            continue
        best = None
        for k, (w, d) in enumerate(zip(wv, dl)):
            if d == 0.0:
                continue
            r = max(abs(F(g[0]) - w[0]), abs(F(g[1]) - w[1])) / F(d)
            if best is None or r < best[0]:
                best = (r, k)
        assert best is not None and best[0] <= 1, (c[4], g, best)
        WORST["ratio"] = max(WORST["ratio"], float(best[0]))
        matched.add(best[1])
    for k, (w, d) in enumerate(zip(wv, dl)):
        if d == 0.0:
            ok = (float(w[0]), float(w[1])) in gv
        else:
            ok = k in matched or any(max(abs(F(g[0]) - w[0]), abs(F(g[1]) - w[1])) <= d for g in gv)
        if not ok:  # collapsed: another referee vertex within rounding distance absorbed it
            assert any(j != k and max(abs(wv[j][0] - w[0]), abs(wv[j][1] - w[1])) <= d + dl[j] + 2 * ulp(cmax) for j in range(len(wv))), (c[4], w)
    dmax = max(dl, default=0.0) or 2 * ulp(cmax)
    err = abs(exact_area(got) - br.area(want))
    assert err <= F(max(perimeter(got), perimeter(br.as_float(want)))) * F(dmax), (c[4], float(err), dmax)


def referee(cases, op):
    return [br.boolean_op(*mem(c), op) for c in cases]


def check_family(ctx, cases, label):
    """the intersection_area and boolean_op checks shared by BA (origin), BB and BC"""
    v = areas(ctx, cases)
    assert np.all(v >= 0.0), label
    for c, x in zip(cases, v):
        a, b = mem(c)
        assert abs(x - float(ov.intersection_area(a, b))) <= tol(a, b), (c[4], x)
        if not pr.intersects(c[1], c[3], c[0], c[2]):
            assert x == 0.0, (c[4], x)
    out = {}
    for op in BF.OPS:
        res = ops_codes(ctx, cases, op)
        want = referee(cases, op)
        for c, (g, code), w in zip(cases, res, want):
            assert code == 0, (label, op, c[4], code, g)
            assert vr.validity_code("multipolygon", g) == 0, (label, op, c[4], g)
            check_geometry(c, g, w)
        out[op] = [g for g, _ in res]
    print(f"{label}: {len(cases)} rows, largest |Δ|/δ so far {WORST['ratio']:.3g}")
    return v, out


def test_ba_origin_and_translations(ctx):
    base, moved = BF.family_ba()
    v0, g0 = check_family(ctx, base, "BA origin")
    inputs = [{(float(x), float(y)) for m in mem(c) for poly in m for r in poly for x, y in r} for c in base]
    for (ox, oy), cases in moved.items():
        v = areas(ctx, cases)
        assert np.array_equal(v.view(np.uint64), v0.view(np.uint64)), (ox, oy)
        for op in BF.OPS:
            g = ops(ctx, cases, op)
            for i, (c, x, x0) in enumerate(zip(cases, g, g0[op])):
                assert [len(m) for m in x] == [len(m) for m in x0], (op, c[4], ox, oy)
                for m, m0 in zip(x, x0):
                    for r, r0 in zip(m, m0):
                        if len(r) != len(r0):  # only where two origin points lie within an ulp at the offset
                            u = ulp(abs(ox) + abs(oy) + 1024)
                            assert any(abs(p[0] - q[0]) <= u and abs(p[1] - q[1]) <= u for p, q in zip(r0[:-1], r0[1:])), (op, c[4])
                            continue
                        for p, p0 in zip(r, r0):
                            if p0 in inputs[i]:
                                assert p == (p0[0] + ox, p0[1] + oy), (op, c[4], p, p0)
                            else:
                                assert abs(p[0] - (p0[0] + ox)) <= ulp(p[0]) and abs(p[1] - (p0[1] + oy)) <= ulp(p[1]), (op, c[4], p, p0)


def test_bb_ulp_gaps(ctx):
    cases = BF.family_bb()
    v, g = check_family(ctx, cases, "BB")
    # the join reproduces the row-wise area and intersection of every pair
    for (ka, kb) in {(c[0], c[2]) for c in cases}:
        sel = [c for c in cases if (c[0], c[2]) == (ka, kb)]
        da = ctx.upload(GeoArrowArray.from_shapes(T[ka], [c[1] for c in sel]))
        db = ctx.upload(GeoArrowArray.from_shapes(T[kb], [c[3] for c in sel]))
        check_joins(ctx, da, db)


def check_joins(ctx, da, db):
    al, ar, area = engine.overlay_area_join(da, db)
    w, _ = engine.intersection_area(ctx.upload(gather(da.to_host(), al)), ctx.upload(gather(db.to_host(), ar)))
    assert np.array_equal(w.view(np.uint64), area.view(np.uint64))
    li, ri, gj = engine.overlay_join(da, db)
    rw = rows(engine.boolean_op(ctx.upload(gather(da.to_host(), li)), ctx.upload(gather(db.to_host(), ri)), "intersection"))
    assert rows(gj) == rw


def test_bc_ring_lengths(ctx):
    closed, unclosed = BF.family_bc()
    check_family(ctx, closed, "BC")
    v0, v1 = areas(ctx, closed), areas(ctx, unclosed)
    assert np.array_equal(v0.view(np.uint64), v1.view(np.uint64))
    for op in BF.OPS:
        assert ops(ctx, unclosed, op) == ops(ctx, closed, op), op


def test_bd_closed_forms(ctx):
    cases = BF.family_bd()
    v = areas(ctx, cases)
    for c, x in zip(cases, v):
        assert abs(x - c[6]) <= tol(*mem(c)), (c[4], x, c[6])
    for op in BF.OPS:
        got = ops(ctx, cases, op)
        for c, g in zip(cases, got):
            assert g == [[[tuple(p) for p in r] for r in m] for m in c[5][op]], (op, c[4])
    for c in cases:
        check_joins(ctx, ctx.upload(GeoArrowArray.from_shapes(T[c[0]], [c[1]])), ctx.upload(GeoArrowArray.from_shapes(T[c[2]], [c[3]])))


def test_is_valid_on_rounded_referee_outputs(ctx):
    """spikes and pinches at 10⁷: the referee's exact rings of BB rounded to doubles, compared code for code"""
    cases = BF.family_bb()
    rounded = [br.as_float(w) for op in BF.OPS for w in referee(cases, op)]
    rounded = [r for r in rounded if r]
    want = [vr.validity_code("multipolygon", r) for r in rounded]
    reason, valid = engine.is_valid(ctx.upload(GeoArrowArray.from_shapes(GeometryType.MULTIPOLYGON, rounded)))
    assert valid.all()
    assert reason.tolist() == want
    assert sum(1 for w in want if w) >= 100
