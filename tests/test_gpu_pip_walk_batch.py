"""The batched walk of the points-in-polygons stream kernel (k_pip_stream<LEAN>, walk_batch in geopolars_b200/csrc/k_pip.cu),
bit-exact against the CPU oracle (`contains_join`, exact orient2d) in the cases the batching adds: batches whose 32 points
all take the longest list a part may have, batches mixing lists without overflow, long overflow runs, cells with several
candidates (the per-point walk) and deferred points, the final partial batch at every queue length, null rows, and
batches whose rows come from several tiles.

Every index here holds plain polygons with FP32 lists only, so the join runs the LEAN kernel; each test asserts it."""
import numpy as np
import pytest

from geopolars_b200 import GeoArrowArray

pytestmark = pytest.mark.gpu

MAX_COUNT = 120  # kFastMaxCount: the longest bucket list a part with FP32 lists may have
FAST_BIT = 1 << 30  # PartLite::nb_flags: the cell record points at the FP32 lists


def fan(x0, y0, w, h, n_edges):
    """a closed (self-crossing) ring of n_edges (even) edges between the bottom and the top of its box, each from the left
    half to the right half: every edge spans the full height and crosses the middle of the x-range, so every y-bucket
    lists every edge, on both sides.  The edges fill an hourglass about the box's centre."""
    m = n_edges // 2
    i = np.arange(m)
    left = np.stack([x0 + i * (0.45 * w / m), np.full(m, y0)], 1)
    right = np.stack([x0 + w - i * (0.45 * w / m), np.full(m, y0 + h)], 1)
    ring = np.empty((2 * m, 2))
    ring[0::2], ring[1::2] = left, right
    return np.concatenate([ring, ring[:1]])


def square(x0, y0, s):
    return np.array([(x0, y0), (x0 + s, y0), (x0 + s, y0 + s), (x0, y0 + s), (x0, y0)], float)


def triangle(x0, y0, s):
    return np.array([(x0, y0), (x0 + s, y0 + 0.3 * s), (x0 + 0.4 * s, y0 + s), (x0, y0)], float)


def polygons(rings):
    xy = np.concatenate(rings)
    ring_off = np.concatenate([[0], np.cumsum([len(r) for r in rings])]).astype(np.int64)
    return GeoArrowArray.polygons(xy, ring_off, np.arange(len(rings) + 1, dtype=np.int64))


def mixed_set():
    """16 polygons on a 4 x 4 layout of 10-unit cells (one per coarse cell of the index, which has 4 per axis), one cell
    holding two overlapping polygons and one left empty: a fan with the longest lists, fans with overflow runs of every
    length, lists without overflow, and a coarse cell with two candidates"""
    c = lambda i: 10.0 * i + 1.0  # noqa: E731
    rings = [fan(c(0), c(0), 8, 8, MAX_COUNT), fan(c(1), c(0), 8, 8, 40), fan(c(2), c(0), 8, 8, 20), triangle(c(3), c(0), 8),
             square(c(0), c(1), 8), fan(c(1), c(1), 8, 8, 16), square(c(1) + 1, c(1) + 1, 6), fan(c(2), c(1), 8, 8, 100),
             fan(c(3), c(1), 8, 8, 4), triangle(c(0), c(2), 8), fan(c(1), c(2), 8, 8, 12), fan(c(2), c(2), 8, 8, 60),
             fan(c(3), c(2), 8, 8, 30), fan(c(0), c(3), 8, 8, 10), fan(c(1), c(3), 8, 8, 80), square(c(3), c(3), 8)]
    return polygons(rings)


def boundary_points(polys, rng, n):
    """vertices and edge midpoints (on the boundary: the FP32 filter cannot certify them) and points 1e-3 off edges"""
    xy = polys.xy
    mid = 0.5 * (xy[:-1] + xy[1:])
    off = xy[:-1] + rng.uniform(0.1, 0.9, (len(xy) - 1, 1)) * (xy[1:] - xy[:-1]) + rng.uniform(-1e-3, 1e-3, (len(xy) - 1, 2))
    pool = np.concatenate([xy, mid, off])
    return pool[rng.integers(0, len(pool), n)]


def walks(idx, polys, pts):
    """which points the stream kernel queues for the walk: inside the union box, in a fine cell of raster code 3 (the
    kernel's fine_index and the raster words of PipIndex.dump)"""
    fg = idx.stats()["fine_cells_per_axis"]
    (x0, y0), (x1, y1) = polys.xy.min(0), polys.xy.max(0)
    px, py = pts[:, 0], pts[:, 1]
    ok = (px >= x0) & (px <= x1) & (py >= y0) & (py <= y1)
    fx = np.clip(np.floor((np.where(ok, px, x0) - x0) * (fg / (x1 - x0))), 0, fg - 1).astype(np.int64)
    fy = np.clip(np.floor((np.where(ok, py, y0) - y0) * (fg / (y1 - y0))), 0, fg - 1).astype(np.int64)
    words = idx.dump("raster").view(np.uint32).reshape(fg, -1, 2)[:, :, 0]
    code = (words[fy, fx >> 4] >> (2 * (fx & 15)).astype(np.uint32)) & 3
    return ok & (code == 3)


def cell_census(idx):
    """(cells with one candidate that has FP32 lists, cells with several candidates)"""
    cells = idx.dump("cells").view(np.int32).reshape(-1, 8)
    return int(((cells[:, 0] == 1) & ((cells[:, 6] & FAST_BIT) != 0)).sum()), int((cells[:, 0] > 1).sum())


def lean_index(ctx, polys):
    from geopolars_b200.engine import PipIndex

    idx = PipIndex(ctx.upload(polys))
    assert idx.stats()["parts_not_fast"] == 0  # every part has FP32 lists and none has holes: the LEAN kernel
    return idx


@pytest.fixture(scope="module")
def mixed(ctx):
    polys = mixed_set()
    idx = lean_index(ctx, polys)
    fast1, multi = cell_census(idx)
    assert fast1 >= 14 and multi >= 1  # lone candidates (batched) and a cell with two (the per-point walk)
    return polys, idx


def test_every_point_takes_the_longest_list(ctx, og, conv):
    """one fan whose every y-bucket lists kFastMaxCount edges on both sides: every walked point reads a list with an
    overflow run of kFastMaxCount - 5 records"""
    polys = polygons([fan(0.0, 0.0, 10.0, 10.0, MAX_COUNT)])
    idx = lean_index(ctx, polys)
    rng = np.random.default_rng(1)
    pts = np.concatenate([rng.uniform(0.0, 10.0, (400_000, 2)), boundary_points(polys, rng, 2_000)])
    w = walks(idx, polys, pts)
    assert w.mean() > 0.3
    pts = pts[w]  # every point walks
    want, wcnt = og.contains_join(conv(polys), pts, use_grid=True, threads=0)
    assert 0 < (want >= 0).sum() < len(pts)
    first, cnt = idx.query(pts, with_count=True)
    assert np.array_equal(first, want) and np.array_equal(cnt, wcnt)


def test_mixed_batches_with_deferred_points(ctx, og, conv, mixed):
    polys, idx = mixed
    rng = np.random.default_rng(2)
    pts = np.concatenate([rng.uniform(0.0, 40.0, (300_000, 2)), boundary_points(polys, rng, 20_000)])
    rng.shuffle(pts)
    want, wcnt = og.contains_join(conv(polys), pts, use_grid=True, threads=0)
    before = idx.stats()["deferred"]
    first, cnt = idx.query(pts, with_count=True)
    assert idx.stats()["deferred"] > before  # points the FP32 filter could not certify went to the exact kernel
    assert np.array_equal(first, want) and np.array_equal(cnt, wcnt)
    assert np.array_equal(idx.query(pts), want)  # ids only


@pytest.mark.parametrize("walked", range(1, 34))
def test_final_partial_batch(ctx, og, conv, mixed, walked):
    """one tile of 100 points, `walked` of them queued: the warp walks a partial batch of `walked` points at the end (one
    full batch first from 32 on)"""
    polys, idx = mixed
    rng = np.random.default_rng(100 + walked)
    pool = np.concatenate([rng.uniform(0.0, 40.0, (4_000, 2)), boundary_points(polys, rng, 1_000)])
    pool = pool[walks(idx, polys, pool)]
    outside = rng.uniform(41.0, 50.0, (100 - walked, 2))
    pts = np.concatenate([pool[rng.choice(len(pool), walked, replace=False)], outside])
    rng.shuffle(pts)
    assert walks(idx, polys, pts).sum() == walked
    want, wcnt = og.contains_join(conv(polys), pts, use_grid=True, threads=0)
    first, cnt = idx.query(pts, with_count=True)
    assert np.array_equal(first, want) and np.array_equal(cnt, wcnt)


def test_null_rows(ctx, og, conv, mixed):
    polys, idx = mixed
    rng = np.random.default_rng(3)
    n = 100_003
    pts = np.concatenate([rng.uniform(0.0, 40.0, (n - 10_000, 2)), boundary_points(polys, rng, 10_000)])
    rng.shuffle(pts)
    valid = rng.random(n) > 0.25
    want, wcnt = og.contains_join(conv(polys), pts, use_grid=True, threads=0)
    assert ((want >= 0) & ~valid).sum() > 1000  # null rows that would match from their coordinates
    first, cnt = idx.query_array(ctx.upload(GeoArrowArray.points(pts, valid=valid)), with_count=True)
    assert np.array_equal(first, np.where(valid, want, -1)) and np.array_equal(cnt, np.where(valid, wcnt, 0))


def test_batches_straddle_tiles(ctx, og, conv, mixed):
    """more tiles of 128 points than resident warps: a warp's queue carries points of one tile into the batches of the
    next, and its last tile is partial"""
    polys, idx = mixed
    rng = np.random.default_rng(4)
    n = 1_000_003
    pts = np.concatenate([rng.uniform(0.0, 40.0, (n - 50_000, 2)), boundary_points(polys, rng, 50_000)])
    rng.shuffle(pts)
    w = walks(idx, polys, pts)
    assert 0.05 < w.mean() < 0.95
    want, wcnt = og.contains_join(conv(polys), pts, use_grid=True, threads=0)
    first, cnt = idx.query(pts, with_count=True)
    assert np.array_equal(first, want) and np.array_equal(cnt, wcnt)
