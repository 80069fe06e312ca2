"""The points-in-polygons join in every index regime, kernel variant and entry point it can take, bit-exact against the CPU
oracle (`contains_join`, exact orient2d; null rows -1 and count 0).

A. Index regimes reached by real inputs: the raster resolution rs falls from 7 to 1 as the polygon count grows (a budget of
   32 M fine cells, G = ceil(sqrt(P)) coarse cells per axis).  Below rs = 4 one raster word spans several coarse cells, so
   stage 2 of the streaming kernel takes candidate #0 from cand01; with G odd the last word of a row is only partly used;
   from 4.19 M parts G is capped at 2048 and coarse cells hold several parts.
B. Kernel variants: the A/B switches are read once per process, so every variant runs in a child process
   (pip_variant_child.py) that writes its outputs to a directory and exits before they are compared.
C. Entry points: null rows in a Point column, the pipelined host path, the per-polygon histograms, more than 2^31 points.

Every test asserts the regime it reached, or the observable effect of its switch, so that a change of the budget or of the
grid cannot make it vacuous."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from geopolars_b200 import GeoArrowArray, GeometryType, synth

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))


# ---- deterministic polygon generator ------------------------------------------------------------------------------------
def star_field(P, holes=True, big=True, seed=0, multi=False):
    """P star polygons of 5-9 vertices on a jittered ceil(sqrt(P))-wide lattice of unit cells, radii up to 0.7 of a cell
    (neighbours overlap); every 97th one spans about 20 cells (long candidate lists), every 89th has a hole (holes=True).
    multi=True: the same parts as MULTIPOLYGON rows of two parts each (the last row may have one)."""
    rng = np.random.default_rng(seed)
    L = int(np.ceil(np.sqrt(P)))
    j = np.arange(P)
    nv = 5 + (j * 7 + seed) % 5
    rmax = np.where(big & (j % 97 == 13), 10.0, 0.7)
    cx = (j % L) + 0.5 + rng.uniform(-0.15, 0.15, P)
    cy = (j // L) + 0.5 + rng.uniform(-0.15, 0.15, P)
    K = 10  # up to 9 vertices + the closing one
    k = np.arange(K)
    th = 2.0 * np.pi * (k[None, :] + rng.uniform(0, 1, P)[:, None]) / nv[:, None]
    r = rmax[:, None] * rng.uniform(0.35, 1.0, (P, K))
    ext = np.stack([cx[:, None] + r * np.cos(th), cy[:, None] + r * np.sin(th)], -1)
    ext[j, nv] = ext[:, 0]  # explicitly closed
    # the star is star-shaped around its centre with every vertex at >= 0.35 rmax: a hole of radius 0.2 rmax stays inside
    has_hole = holes & (j % 89 == 7)
    hk = np.arange(5)
    hth = -2.0 * np.pi * (hk % 4) / 4.0  # clockwise square, closed
    hole = np.stack([cx[:, None] + 0.2 * rmax[:, None] * np.cos(hth)[None, :], cy[:, None] + 0.2 * rmax[:, None] * np.sin(hth)[None, :]], -1)
    coords = np.concatenate([ext, hole], 1)
    keep = np.concatenate([k[None, :] <= nv[:, None], np.broadcast_to(has_hole[:, None], (P, 5))], 1)
    xy = coords[keep]
    ring_len = np.stack([nv + 1, np.where(has_hole, 5, 0)], 1)
    lens = ring_len[np.stack([np.ones(P, bool), has_hole], 1)]
    ring_off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    part_off = np.concatenate([[0], np.cumsum(1 + has_hole)]).astype(np.int64)
    if not multi:
        return GeoArrowArray.polygons(xy, ring_off, part_off)
    geom_off = np.concatenate([np.arange(0, P, 2), [P]]).astype(np.int64)
    return GeoArrowArray.multipolygons(xy, ring_off, part_off, geom_off)


def field_points(polys, n, seed=0, every=50, cap=100_000):
    """n uniform points over the union box plus a margin; every `every`-th vertex and edge midpoint, each also one ulp
    either way; NaN and +-inf coordinates"""
    rng = np.random.default_rng(1000 + seed)
    xy = polys.xy
    lo, hi = xy.min(0), xy.max(0)
    m = 0.02 * (hi - lo) + 1e-3
    uni = rng.uniform(lo - m, hi + m, (n, 2))
    v = xy[::every][:cap]
    mid = (0.5 * (xy[:-1] + xy[1:]))[::every][:cap]
    spec = np.concatenate([v, mid])
    c = 0.5 * (lo + hi)
    inf, nan = np.inf, np.nan
    odd = np.array([[nan, c[1]], [c[0], nan], [nan, nan], [inf, c[1]], [-inf, c[1]], [c[0], inf], [c[0], -inf], [inf, inf], [-inf, -inf]])
    return np.concatenate([uni, spec, np.nextafter(spec, np.inf), np.nextafter(spec, -np.inf), odd])


def lattice_points(polys, fg, step=13, rows=200):
    """points ON the fine-cell lattice of the union box (as the index computes it), each also one ulp either way"""
    ext = polys.xy  # holes lie inside their exteriors: the union box of every coordinate is the index's
    x0, y0 = ext.min(0)
    w, h = ext.max(0) - (x0, y0)
    k = np.arange(0, fg + 1, step, dtype=np.float64)
    gx, gy = np.meshgrid(x0 + k / fg * w, y0 + (k[:rows] + 3) / fg * h)
    lat = np.stack([gx.ravel(), gy.ravel()], 1)
    return np.concatenate([lat, np.nextafter(lat, np.inf), np.nextafter(lat, -np.inf)])


def rows_rings(a, row):
    """the parts of one row as lists of rings of (x, y) tuples (oracle/exact.py's input)"""
    if a.type == GeometryType.POLYGON:
        parts = [(a.geom_off[row], a.geom_off[row + 1])]
    else:
        parts = [(a.part_off[p], a.part_off[p + 1]) for p in range(a.geom_off[row], a.geom_off[row + 1])]
    return [[[tuple(c) for c in a.xy[a.ring_off[r]:a.ring_off[r + 1]]] for r in range(r0, r1)] for r0, r1 in parts]


def row_boxes(a):
    """(n_rows, 4) envelope xmin, ymin, xmax, ymax of every row (exterior rings; holes lie inside)"""
    ring_row = np.repeat(np.arange(a.n_rings), np.diff(a.ring_off))
    if a.type == GeometryType.POLYGON:
        row_of_ring = np.repeat(np.arange(len(a)), np.diff(a.geom_off))
    else:
        part_row = np.repeat(np.arange(len(a)), np.diff(a.geom_off))
        row_of_ring = part_row[np.repeat(np.arange(a.n_parts), np.diff(a.part_off))]
    row = row_of_ring[ring_row]
    box = np.empty((len(a), 4))
    box[:, :2], box[:, 2:] = np.inf, -np.inf
    np.minimum.at(box[:, 0], row, a.xy[:, 0])
    np.minimum.at(box[:, 1], row, a.xy[:, 1])
    np.maximum.at(box[:, 2], row, a.xy[:, 0])
    np.maximum.at(box[:, 3], row, a.xy[:, 1])
    return box


def check_pairs(lhs, rhs, want, wcnt):
    """pair list sorted by point: every point once per containing row, rows ascending, the first one the oracle's"""
    lhs, rhs = lhs.astype(np.int64), rhs.astype(np.int64)
    assert np.array_equal(lhs, np.repeat(np.arange(len(want)), wcnt))
    starts = np.concatenate([[0], np.cumsum(wcnt)[:-1]])
    hit = wcnt > 0
    assert np.array_equal(rhs[starts[hit]], want[hit])
    same = lhs[1:] == lhs[:-1]
    assert (rhs[1:][same] > rhs[:-1][same]).all()


def exact_cross_check(polys, pts, want, wcnt, boxes):
    """the oracle against oracle/exact.py (rational arithmetic) with candidates found by envelope on the host"""
    from oracle import exact

    for (x, y), f, c in zip(pts, want, wcnt):
        if not (np.isfinite(x) and np.isfinite(y)):
            assert f == -1 and c == 0
            continue
        cand = np.nonzero((boxes[:, 0] <= x) & (x <= boxes[:, 2]) & (boxes[:, 1] <= y) & (y <= boxes[:, 3]))[0]
        rows = [int(r) for r in cand if any(exact.polygon_contains((float(x), float(y)), part) for part in rows_rings(polys, r))]
        assert (f, c) == ((rows[0] if rows else -1), len(rows)), (x, y, f, c, rows)


def expected_grid(P, mcells=32, rs_max=7):
    G = min(2048, max(1, int(np.ceil(np.sqrt(P)))))
    rs = rs_max
    while rs > 0 and ((G << rs) > (1 << 20) or (G << rs) ** 2 > (mcells << 20)):
        rs -= 1
    return G, rs


# ---- A. index regimes -----------------------------------------------------------------------------------------------------
REGIMES = [
    # (form, polygons, rs, G)
    ("polygon", 151_000, 3, 389),
    ("polygon", 600_000, 2, 775),
    ("polygon", 2_200_000, 1, 1484),
    ("polygon", 5_000_000, 1, 2048),
    ("polygon-holes", 151_000, 3, 389),
    ("multipolygon", 151_000, 3, 389),
]


@pytest.mark.parametrize("form,P,rs,G", REGIMES, ids=[f"{f}-{p}" for f, p, _, _ in REGIMES])
def test_index_regimes_vs_oracle(ctx, og, conv, form, P, rs, G):
    """coarse rasters (rs < 4: raster words span several coarse cells), partly used last raster words (G << rs not a multiple
    of 16), and G capped at 2048 (more parts than coarse cells); LEAN on plain POLYGON rows, the full walk with holes and on
    MULTIPOLYGON rows"""
    from geopolars_b200.engine import PipIndex

    polys = star_field(P, holes=form != "polygon", seed=P % 1000, multi=form == "multipolygon")
    assert expected_grid(P) == (G, rs)
    idx = PipIndex(ctx.upload(polys))
    st = idx.stats()
    fg = st["fine_cells_per_axis"]
    assert (st["raster_log2"], st["coarse_cells_per_axis"], fg) == (rs, G, G << rs), st
    assert (fg % 16 != 0) == (P != 5_000_000)  # the partial last word of every raster row
    total = fg * fg
    assert 0.01 * total < st["raster_walk_cells"] < total, st
    assert st["raster_inside_cells"] > 0.001 * total, st  # some points are answered from the raster (codes 1 and 2)
    boxes = row_boxes(polys)
    if P == 5_000_000:  # more parts than coarse cells: the candidate lists of most cells are long
        x0, y0 = polys.xy.min(0)
        x1, y1 = polys.xy.max(0)
        inv_w, inv_h = fg / (x1 - x0), fg / (y1 - y0)
        cx = [np.clip(np.floor((boxes[:, k] - x0) * inv_w), 0, fg - 1).astype(np.int64) >> rs for k in (0, 2)]
        cy = [np.clip(np.floor((boxes[:, k] - y0) * inv_h), 0, fg - 1).astype(np.int64) >> rs for k in (1, 3)]
        d = np.zeros((G + 1, G + 1), np.int64)  # 2-D difference array of the envelopes' cell ranges
        np.add.at(d, (cy[0], cx[0]), 1)
        np.add.at(d, (cy[0], cx[1] + 1), -1)
        np.add.at(d, (cy[1] + 1, cx[0]), -1)
        np.add.at(d, (cy[1] + 1, cx[1] + 1), 1)
        per_cell = d.cumsum(0).cumsum(1)[:G, :G]
        assert (per_cell >= 2).mean() > 0.5 and (per_cell >= 3).mean() > 0.2, ((per_cell >= 2).mean(), (per_cell >= 3).mean())

    base = field_points(polys, 1_700_000, seed=P % 7, every=50, cap=60_000)
    pts = np.concatenate([base, lattice_points(polys, fg)])
    want, wcnt = og.contains_join(conv(polys), pts, use_grid=True, threads=0)
    assert 0 < (want >= 0).sum() < len(pts) and wcnt.max() >= 2
    first, cnt = idx.query(pts, with_count=True)
    assert np.array_equal(first, want), np.nonzero(first != want)[0][:10]
    assert np.array_equal(cnt, wcnt)
    f2, counts = idx.query_counts(pts)
    assert np.array_equal(f2, want)
    assert np.array_equal(counts.astype(np.int64), np.bincount(want[want >= 0], minlength=len(polys)))
    lhs, rhs = idx.pairs(pts)
    check_pairs(lhs, rhs, want, wcnt)
    # the oracle itself, on boundary and one-ulp points, against exact rational arithmetic
    n_uni = 1_700_000
    sel = np.linspace(n_uni, len(base) - 10, 1800).astype(np.int64)
    sel = np.concatenate([sel, np.arange(len(base) - 9, len(base)), len(base) + np.arange(0, 3 * 9000, 137)[:200]])
    exact_cross_check(polys, pts[sel], want[sel], wcnt[sel], boxes)


# ---- B. kernel variants in child processes ----------------------------------------------------------------------------------
VARIANTS = {
    "default": {},
    "lean0": {"GPL_PIP_LEAN": "0"},
    "legacy": {"GPL_PIP_LEGACY": "1"},
    "legacy-lean0": {"GPL_PIP_LEGACY": "1", "GPL_PIP_LEAN": "0"},
    "cand-smem": {"GPL_PIP_CAND_SMEM": "1"},
    "fuse-hist": {"GPL_PIP_FUSE_HIST": "1"},
    **{f"ld-hints{h}": {"GPL_PIP_LD_HINTS": str(h)} for h in (0, 1, 2, 3, 4, 6, 7)},
    "one-cta-per-sm": {"GPL_PIP_STREAM_CTAS_PER_SM": "1", "GPL_PIP_CTAS_PER_SM": "1"},
    **{f"raster-log2-{k}": {"GPL_PIP_RASTER_LOG2": str(k)} for k in (0, 1, 2, 3)},
    "raster-1mcells": {"GPL_PIP_RASTER_MCELLS": "1"},
    "slots-25": {"GPL_PIP_SLOTS_X100": "25"},
    "slots-6400": {"GPL_PIP_SLOTS_X100": "6400"},
    "no-l2-pin": {"GPL_L2_PIN": "0"},
}
_SWITCHES = sorted({k for v in VARIANTS.values() for k in v} | {"GPL_PIP_LEAN_CTAS_PER_SM", "GPL_PIP_NOALLOC"})


def run_variant(tmp_path_factory, name):
    out = tmp_path_factory.mktemp("pip-" + name)
    env = {k: v for k, v in os.environ.items() if k not in _SWITCHES}
    env.update(VARIANTS[name])
    subprocess.run([sys.executable, os.path.join(HERE, "pip_variant_child.py"), str(out)], env=env, timeout=900, check=True)
    with open(out / "meta.json") as f:
        meta = json.load(f)
    return {k: dict(np.load(out / f"{k}.npz")) for k in meta}, meta


@pytest.fixture(scope="module")
def variant_oracle(og, conv):
    import pip_variant_child as child

    out = {}
    for name, (polys, pts) in child.cases().items():
        want, wcnt = og.contains_join(conv(polys), pts, use_grid=True, threads=0)
        valid = child.null_mask(len(pts))
        out[name] = dict(n_geoms=len(polys), want=want, wcnt=wcnt, want_v=np.where(valid, want, -1), wcnt_v=np.where(valid, wcnt, 0))
    return out


@pytest.fixture(scope="module")
def control(tmp_path_factory):
    return run_variant(tmp_path_factory, "default")


@pytest.mark.parametrize("variant", list(VARIANTS))
def test_kernel_variants_vs_oracle(variant, variant_oracle, control, tmp_path_factory):
    """every entry point under every A/B switch.  Where the ABI shows the path taken, the test asserts it: raster_log2 and
    fine_cells_per_axis for the raster switches, the index bytes for the bucket sizing, one launch fewer for query_counts
    with fused bins, no kernel-timing pair for the round-1 kernel.  Nothing in the ABI shows whether the LEAN walk, the
    shared-memory candidate rows or a cache-hint variant ran; those variants are checked on their outputs only."""
    res, meta = control if variant == "default" else run_variant(tmp_path_factory, variant)
    _, cmeta = control
    for name, o in variant_oracle.items():
        r, st, cst = res[name], meta[name]["stats"], cmeta[name]["stats"]
        want, wcnt = o["want"], o["wcnt"]
        for k, (f, c) in {"query": ("q_first", "q_cnt"), "device": ("d_first", "d_cnt")}.items():
            assert np.array_equal(r[f], want), (name, k, np.nonzero(r[f] != want)[0][:10])
            assert np.array_equal(r[c], wcnt), (name, k)
        assert np.array_equal(r["q_only"], want), name
        assert np.array_equal(r["c_first"], want), name
        assert np.array_equal(r["c_counts"].astype(np.int64), np.bincount(want[want >= 0], minlength=o["n_geoms"])), name
        check_pairs(r["p_lhs"], r["p_rhs"], want, wcnt)
        assert np.array_equal(r["a_first"], o["want_v"]), (name, np.nonzero(r["a_first"] != o["want_v"])[0][:10])
        assert np.array_equal(r["a_cnt"], o["wcnt_v"]), name
        check_pairs(r["pa_lhs"], r["pa_rhs"], o["want_v"], o["wcnt_v"])
        # the switch took effect
        env = VARIANTS[variant]
        G = cst["coarse_cells_per_axis"]
        assert st["coarse_cells_per_axis"] == G and st["fine_cells_per_axis"] == G << st["raster_log2"]
        if "GPL_PIP_RASTER_LOG2" in env:
            assert st["raster_log2"] == min(int(env["GPL_PIP_RASTER_LOG2"]), cst["raster_log2"]), (name, st)
        elif "GPL_PIP_RASTER_MCELLS" in env:
            assert st["raster_log2"] == expected_grid(G * G, mcells=1)[1] <= cst["raster_log2"], (name, st)
        else:
            assert st["raster_log2"] == cst["raster_log2"], (name, st)
        if env.get("GPL_PIP_SLOTS_X100") == "25":
            assert st["bytes"] > cst["bytes"], (name, st["bytes"], cst["bytes"])
        elif env.get("GPL_PIP_SLOTS_X100") == "6400":
            assert st["bytes"] <= cst["bytes"] and (st["bytes"] < cst["bytes"] or name in ("one", "holes_multis")), (name, st["bytes"])
        elif st["raster_log2"] == cst["raster_log2"]:
            assert st["bytes"] == cst["bytes"], name
        fused = variant == "fuse-hist" and o["n_geoms"] <= 12288
        assert meta[name]["launches_counts"] == cmeta[name]["launches_counts"] - int(fused), (name, meta[name], cmeta[name])
        legacy = "GPL_PIP_LEGACY" in env
        assert meta[name]["timed_stream_launches"] == (0 if legacy else 1), (name, meta[name])
    if variant == "fuse-hist":
        assert any(o["n_geoms"] <= 12288 for o in variant_oracle.values())
    if "GPL_PIP_RASTER_MCELLS" in VARIANTS[variant]:  # the budget, not the 2^7 cap, set the resolution somewhere
        assert any(meta[k]["stats"]["raster_log2"] < cmeta[k]["stats"]["raster_log2"] for k in meta)


# ---- C. entry points ------------------------------------------------------------------------------------------------------
def test_null_points_with_coordinates_inside_polygons(ctx, og, conv):
    """a Point column with a validity bitmap whose null rows hold coordinates inside polygons and on their boundaries: the
    count pass and the pair kernel must both skip them (otherwise the pair kernel writes outside its slot in the scan)"""
    from geopolars_b200 import geoseries as gs
    from geopolars_b200.engine import PipIndex

    polys = star_field(2500, holes=True, seed=5)
    n = 100_003
    assert n % 8 != 0
    rng = np.random.default_rng(9)
    ctr = 0.5 * (polys.xy[polys.ring_off[polys.geom_off[:-1]]] + polys.xy[polys.ring_off[polys.geom_off[:-1]] + 2])
    pts = np.concatenate([ctr[rng.integers(0, len(ctr), n // 2)], polys.xy[rng.integers(0, polys.n_coords, n - n // 2)]])
    rng.shuffle(pts)
    valid = np.ones(n, bool)
    valid[rng.integers(0, n, n // 4)] = False
    valid[[0, 127, 128, 129, n - 1]] = False
    want, wcnt = og.contains_join(conv(polys), pts, use_grid=True, threads=0)
    assert (want[~valid] >= 0).sum() > 1000  # null rows that WOULD be matched from their coordinates
    want_v, wcnt_v = np.where(valid, want, -1), np.where(valid, wcnt, 0)
    d_pts = ctx.upload(GeoArrowArray.points(pts, valid=valid))
    d_polys = ctx.upload(polys)
    idx = PipIndex(d_polys)
    first, cnt = idx.query_array(d_pts, with_count=True)
    assert np.array_equal(first, want_v) and np.array_equal(cnt, wcnt_v)
    lhs, rhs = idx.pairs_array(d_pts)
    check_pairs(lhs, rhs, want_v, wcnt_v)
    assert not np.isin(lhs.astype(np.int64), np.nonzero(~valid)[0]).any()
    a, b = gs.spatial_join(gs.GeoSeries(_device=d_pts), gs.GeoSeries(_device=d_polys), how="left")
    assert np.array_equal(a, np.repeat(np.arange(n), np.maximum(wcnt_v, 1)))
    assert (b[np.isin(a, np.nonzero(~valid)[0])] == -1).all()
    hit = np.repeat(wcnt_v > 0, np.maximum(wcnt_v, 1))
    assert np.array_equal(b[hit], rhs.astype(np.int64))


def test_pipelined_host_path_chunks_and_buffers(ctx, og, conv):
    """gpl_contains_join_host: ragged tails, a chunk larger than the column, the default chunk, one-point chunks; pageable
    numpy and pinned torch buffers; called while other work is still queued on the context stream"""
    import torch

    from geopolars_b200.engine import PipIndex

    polys = star_field(2500, holes=False, seed=6)
    idx = PipIndex(ctx.upload(polys))
    n = 1_000_003
    pts = field_points(polys, n - 2 * 9 - 9, seed=6, every=40, cap=3)[:n]
    assert len(pts) == n
    want = idx.query(pts)
    assert np.array_equal(want, og.contains_join(conv(polys), pts, use_grid=True, threads=0)[0])
    busy = torch.from_numpy(synth.uniform_points(8_000_000, scale=50.0)).cuda()
    busy_ids = torch.empty(len(busy), dtype=torch.int32, device="cuda")
    t_pts = torch.from_numpy(pts).pin_memory()
    sentinel = -7
    for chunk in (127, 128, 129, 4097, n - 1, n, 2 * n, 0):
        for kind in ("pageable", "pinned"):
            torch.cuda.synchronize()
            idx.query_device(busy.data_ptr(), len(busy), busy_ids.data_ptr())  # queued on the context stream, not waited for
            if kind == "pageable":
                ids = np.full(n + 1, sentinel, np.int32)
                idx.query_host_pipelined(pts.ctypes.data, n, ids.ctypes.data, chunk)
                got = ids
            else:
                ids_t = torch.full((n + 1,), sentinel, dtype=torch.int32).pin_memory()
                idx.query_host_pipelined(t_pts.data_ptr(), n, ids_t.data_ptr(), chunk)
                got = ids_t.numpy()
            assert got[n] == sentinel, (chunk, kind)
            assert np.array_equal(got[:n], want), (chunk, kind, np.nonzero(got[:n] != want)[0][:5])
    small = pts[:5000]
    ids = np.full(5001, sentinel, np.int32)
    idx.query_host_pipelined(small.ctypes.data, 5000, ids.ctypes.data, 1)
    assert ids[5000] == sentinel and np.array_equal(ids[:5000], want[:5000])
    ctx.synchronize()


@pytest.mark.parametrize("P", [1, 12_288, 12_289, 49_152, 49_153, 151_000])
def test_histograms_accumulate_and_take_every_path(ctx, og, conv, P):
    """per-polygon counts: shared-memory bins up to 49 152 polygons, global atomics above; counts accumulate into the
    column they are given; k_histogram's scalar path for id columns that are not 16-byte aligned, its tail, and ids outside
    [0, n_polygons)"""
    import torch

    from geopolars_b200 import engine as E

    polys = star_field(P, holes=False, seed=P % 11) if P > 1 else GeoArrowArray.from_shapes(
        GeometryType.POLYGON, [[[(0.0, 0.0), (4.0, 1.0), (5.0, 5.0), (1.0, 3.5), (0.0, 0.0)]]])
    idx = E.PipIndex(ctx.upload(polys))
    pts = field_points(polys, 300_001, seed=3, every=50, cap=20_000)
    want, _ = og.contains_join(conv(polys), pts, use_grid=True, threads=0)
    hist = np.bincount(want[want >= 0], minlength=P).astype(np.uint64)
    assert hist.sum() > 1000
    start = (np.arange(P, dtype=np.uint64) * 7919 + 3) % 100_003
    # host buffers
    first = np.empty(len(pts), np.int32)
    counts = start.copy()
    E.check(ctx.lib.gpl_contains_join_counts(ctx._h, idx._h, pts.ctypes.data, len(pts), first.ctypes.data, counts.ctypes.data, E.GPL_HOST))
    assert np.array_equal(first, want) and np.array_equal(counts, start + hist)
    # device buffers, twice into the same column
    d_pts = torch.from_numpy(pts).cuda()
    d_first = torch.empty(len(pts), dtype=torch.int32, device="cuda")
    d_counts = torch.from_numpy(start.astype(np.int64)).cuda()
    torch.cuda.synchronize()
    for _ in range(2):
        idx.query_device_counts(d_pts.data_ptr(), len(pts), d_first.data_ptr(), d_counts.data_ptr())
    ctx.synchronize()
    assert np.array_equal(d_first.cpu().numpy(), want)
    assert np.array_equal(d_counts.cpu().numpy().astype(np.uint64), start + 2 * hist)
    # gpl_join_histogram on id columns starting 0..3 elements into an aligned buffer, with -1 and ids >= n_polygons
    ids = np.concatenate([[-1, P, P + 5, -1], want, [P, -1, 2 ** 31 - 1, 0]]).astype(np.int32)
    d_ids = torch.from_numpy(ids).cuda()
    for off in (0, 1, 2, 3):
        col = ids[off:len(ids) - off]
        d_h = torch.from_numpy(start.astype(np.int64)).cuda()
        torch.cuda.synchronize()
        E.check(ctx.lib.gpl_join_histogram(ctx._h, d_ids.data_ptr() + 4 * off, len(col), d_h.data_ptr(), P, E.GPL_DEVICE))
        ctx.synchronize()
        ok = col[(col >= 0) & (col < P)]
        assert np.array_equal(d_h.cpu().numpy().astype(np.uint64), start + np.bincount(ok, minlength=P).astype(np.uint64)), off


def test_more_than_2_31_points_with_nulls(og, conv):
    """pip_query splits at 2^31 points per launch pair: chunk-relative deferred indices, a validity pointer advanced by
    lo / 8, ids and counts written at lo.  n = 2^31 + 2^22 + 5 device points (every 7th row null), outputs on the device."""
    import torch

    from geopolars_b200 import engine as E

    free, _ = torch.cuda.mem_get_info()
    if free < 56 * 2 ** 30:
        pytest.skip(f"needs 56 GB of free device memory, {free / 2 ** 30:.1f} GB free")
    n = 2 ** 31 + 2 ** 22 + 5
    ctx = E.Context(0)
    try:
        xy, ro, go = synth.star_polygons(10_000, 100)
        polys = GeoArrowArray.polygons(xy, ro, go)
        idx = E.PipIndex(ctx.upload(polys))
        pts = torch.empty((n, 2), dtype=torch.float64, device="cuda")
        E.check(ctx.lib.gpl_gen_uniform_points(ctx._h, 2, 0, n, 1000.0, pts.data_ptr()))
        nbytes = (n + 7) // 8
        pattern = np.packbits(np.arange(56) % 7 != 0, bitorder="little")  # 7 bytes: bit i set <=> row i is not a multiple of 7
        bm = torch.from_numpy(pattern).cuda().repeat((nbytes + 6) // 7)[:nbytes].contiguous()
        ctx.synchronize()
        arr = ctx.wrap_device(GeometryType.POINT, n, n, pts.data_ptr(), validity_ptr=bm.data_ptr(), keepalive=(pts, bm))
        ids = torch.empty(n, dtype=torch.int32, device="cuda")
        cnt = torch.empty(n, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        E.check(ctx.lib.gpl_contains_join_array(ctx._h, idx._h, arr._h, C.c_void_p(ids.data_ptr()), C.c_void_p(cnt.data_ptr()), E.GPL_DEVICE))
        ctx.synchronize()
        opolys = conv(polys)
        split = 2 ** 31
        for lo, m in ((0, 16 * 2 ** 20), (split - 8 * 2 ** 20, n - split + 8 * 2 ** 20)):  # the first 16 M rows, the last 12 M
            hp = og.gen_uniform_points(2, lo, m, 1000.0)
            want, wcnt = og.contains_join(opolys, hp, use_grid=True, threads=0)
            null = (np.arange(lo, lo + m) % 7) == 0
            want[null], wcnt[null] = -1, 0
            assert (want >= 0).any()
            assert np.array_equal(ids[lo:lo + m].cpu().numpy(), want), (lo, np.nonzero(ids[lo:lo + m].cpu().numpy() != want)[0][:5])
            assert np.array_equal(cnt[lo:lo + m].cpu().numpy(), wcnt), lo
        del cnt
        counts = torch.zeros(10_000, dtype=torch.int64, device="cuda")
        E.check(ctx.lib.gpl_join_histogram(ctx._h, ids.data_ptr(), n, counts.data_ptr(), 10_000, E.GPL_DEVICE))
        ctx.synchronize()
        ref = torch.zeros(10_000, dtype=torch.int64, device="cuda")
        step = 2 ** 28
        for lo in range(0, n, step):
            c = ids[lo:lo + step]
            ref += torch.bincount(c[c >= 0].long(), minlength=10_000)
        assert torch.equal(counts, ref)
        assert int(ref.sum()) > 0.3 * n * 6 / 7
    finally:
        ctx.close()
