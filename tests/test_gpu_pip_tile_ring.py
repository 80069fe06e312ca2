"""The output path of the points-in-polygons stream kernel (k_pip_stream, geopolars_b200/csrc/k_pip.cu): every warp keeps
its last kRing tiles of ids (and counts) in a ring in shared memory, the walk writes its results there, and a tile is
stored once, as a whole, when its slot is taken again or at the end.  Bit-exact against the CPU oracle, ids only and with
counts, in the cases the ring adds: tiles whose every point walks, tiles with no walker, walkers that wait kRing tiles or
more in the queue (the partial batch before a slot is taken), sizes around a tile and around the ring of every launched
warp, id and count columns that are only 4-byte aligned, null rows and deferred points.

The columns are built point by point from the index's raster (which points the kernel queues for the walk), so each test
controls the walker mix of every tile.  Every index here runs the LEAN kernel, except in test_full_walk_kernel."""
import numpy as np
import pytest

from geopolars_b200 import GeoArrowArray
from test_gpu_pip_regimes import star_field
from test_gpu_pip_walk_batch import boundary_points, lean_index, mixed_set, walks

pytestmark = pytest.mark.gpu

TILE = 128  # kTilePts
RING = 4  # kRing
WARPS = 132 * 3 * 8  # the stream kernel's resident warps on an H100: 132 SMs x 3 CTAs x 8 warps


@pytest.fixture(scope="module")
def mixed(ctx):
    polys = mixed_set()
    idx = lean_index(ctx, polys)
    rng = np.random.default_rng(11)
    pool = np.concatenate([rng.uniform(0.0, 40.0, (400_000, 2)), boundary_points(polys, rng, 40_000)])
    w = walks(idx, polys, pool)
    return polys, idx, pool[w], pool[~w]


def column(rng, walker_pool, still_pool, walk):
    """one point per row: a walker where `walk` is set, a point that does not walk elsewhere"""
    pts = still_pool[rng.integers(0, len(still_pool), len(walk))]
    pts[walk] = walker_pool[rng.integers(0, len(walker_pool), int(walk.sum()))]
    return pts


def per_tile(rng, n, fractions):
    """walker mask of n rows: each tile of 128 rows walks a fraction drawn from `fractions`"""
    f = rng.choice(fractions, -(-n // TILE))
    return rng.random(n) < np.repeat(f, TILE)[:n]


def check_join(og, conv, polys, idx, pts):
    want, wcnt = og.contains_join(conv(polys), pts, use_grid=True, threads=0)
    first, cnt = idx.query(pts, with_count=True)
    assert np.array_equal(first, want) and np.array_equal(cnt, wcnt)
    assert np.array_equal(idx.query(pts), want)
    return want


def test_every_point_walks(ctx, og, conv, mixed):
    """more than kRing tiles per warp, every row a walker: each tile leaves as four full batches"""
    polys, idx, wpool, spool = mixed
    rng = np.random.default_rng(1)
    n = (RING + 2) * WARPS * TILE + 77
    pts = column(rng, wpool, spool, np.ones(n, bool))
    assert walks(idx, polys, pts).all()
    check_join(og, conv, polys, idx, pts)


def test_tiles_without_walkers(ctx, og, conv, mixed):
    """tiles with no walker between tiles where every point walks and tiles with a few"""
    polys, idx, wpool, spool = mixed
    rng = np.random.default_rng(2)
    n = (RING + 3) * WARPS * TILE + 5
    walk = per_tile(rng, n, [0.0, 0.0, 0.05, 1.0])
    pts = column(rng, wpool, spool, walk)
    w = walks(idx, polys, pts)
    tiles = np.add.reduceat(w, np.arange(0, n, TILE))
    assert (tiles == 0).sum() > 1000 and (tiles >= 120).sum() > 1000
    check_join(og, conv, polys, idx, pts)


@pytest.mark.parametrize("per_tile_walkers", [1, 4, 10])
def test_walkers_wait_ring_tiles(ctx, og, conv, mixed, per_tile_walkers):
    """fewer than 32 walkers in any kRing - 1 consecutive tiles of a warp: the queue never fills a batch, and the oldest
    walkers are walked kRing tiles after their own one, in a partial batch, just before their slot is taken"""
    polys, idx, wpool, spool = mixed
    rng = np.random.default_rng(3 + per_tile_walkers)
    n = (3 * RING + 1) * WARPS * TILE
    walk = np.zeros(n, bool)
    rows = np.arange(0, n, TILE)[:, None] + rng.integers(0, TILE, (n // TILE, per_tile_walkers))
    walk[rows.ravel()] = True
    pts = column(rng, wpool, spool, walk)
    w = walks(idx, polys, pts)
    assert np.add.reduceat(w, np.arange(0, n, TILE)).max() <= per_tile_walkers
    check_join(og, conv, polys, idx, pts)


@pytest.mark.parametrize("n", [1, 31, 127, 128, 129, 1_000, 12_345, RING * TILE * WARPS, RING * TILE * WARPS + 1])
def test_sizes(ctx, og, conv, mixed, n):
    """below one tile, not a multiple of a tile, exactly kRing tiles on every resident warp (and one point more)"""
    polys, idx, wpool, spool = mixed
    rng = np.random.default_rng(n)
    pts = column(rng, wpool, spool, rng.random(n) < 0.3)
    check_join(og, conv, polys, idx, pts)


@pytest.mark.parametrize("id_off,cnt_off", [(1, 1), (1, 0), (0, 1), (0, 0)])
def test_id_and_count_columns_offset(ctx, og, conv, mixed, id_off, cnt_off):
    """id and count columns that start 4 bytes past a 16-byte boundary take the per-lane stores of the tile; the rows
    around them stay untouched"""
    import torch

    polys, idx, wpool, spool = mixed
    rng = np.random.default_rng(20 + 2 * id_off + cnt_off)
    n = 2 * WARPS * TILE + 1_001
    pts = column(rng, wpool, spool, per_tile(rng, n, [0.0, 0.2, 1.0]))
    want, wcnt = og.contains_join(conv(polys), pts, use_grid=True, threads=0)
    d_pts = torch.from_numpy(pts).cuda()
    d_ids = torch.full((n + 8,), -7, dtype=torch.int32, device="cuda")
    d_cnt = torch.full((n + 8,), -7, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    idx.query_device(d_pts.data_ptr(), n, d_ids.data_ptr() + 4 * id_off, d_cnt.data_ptr() + 4 * cnt_off)
    ctx.synchronize()
    ids, cnt = d_ids.cpu().numpy(), d_cnt.cpu().numpy()
    assert np.array_equal(ids[id_off:id_off + n], want) and np.array_equal(cnt[cnt_off:cnt_off + n], wcnt)
    assert (ids[:id_off] == -7).all() and (ids[id_off + n:] == -7).all()
    assert (cnt[:cnt_off] == -7).all() and (cnt[cnt_off + n:] == -7).all()
    d_ids.fill_(-7)
    torch.cuda.synchronize()
    idx.query_device(d_pts.data_ptr(), n, d_ids.data_ptr() + 4 * id_off)
    ctx.synchronize()
    ids = d_ids.cpu().numpy()
    assert np.array_equal(ids[id_off:id_off + n], want) and (ids[id_off + n:] == -7).all()


def test_null_rows(ctx, og, conv, mixed):
    polys, idx, wpool, spool = mixed
    rng = np.random.default_rng(4)
    n = (RING + 1) * WARPS * TILE + 3
    pts = column(rng, wpool, spool, per_tile(rng, n, [0.0, 0.1, 1.0]))
    valid = rng.random(n) > 0.3
    want, wcnt = og.contains_join(conv(polys), pts, use_grid=True, threads=0)
    assert ((want >= 0) & ~valid).sum() > 10_000  # null rows that would match from their coordinates
    d = ctx.upload(GeoArrowArray.points(pts, valid=valid))
    first, cnt = idx.query_array(d, with_count=True)
    assert np.array_equal(first, np.where(valid, want, -1)) and np.array_equal(cnt, np.where(valid, wcnt, 0))
    assert np.array_equal(idx.query_array(d), np.where(valid, want, -1))


def test_deferred_points(ctx, og, conv, mixed):
    """points on edges and vertices: the filter defers them, the exact kernel rewrites their ids after the tiles left"""
    polys, idx, wpool, spool = mixed
    rng = np.random.default_rng(5)
    n = (RING + 1) * WARPS * TILE + 9
    pts = column(rng, wpool, spool, per_tile(rng, n, [0.0, 0.1, 1.0]))
    edge = rng.random(n) < 0.02
    pts[edge] = boundary_points(polys, rng, int(edge.sum()))
    before = idx.stats()["deferred"]
    check_join(og, conv, polys, idx, pts)
    assert idx.stats()["deferred"] - before > 1000


@pytest.mark.parametrize("multi", [False, True])
def test_full_walk_kernel(ctx, og, conv, multi):
    """polygons with holes and MULTIPOLYGON rows take the kernel without the LEAN restriction, which keeps the same ring:
    several tiles per warp, ids and counts"""
    from geopolars_b200.engine import PipIndex

    polys = star_field(20_000, holes=True, seed=7, multi=multi)
    idx = PipIndex(ctx.upload(polys))
    rng = np.random.default_rng(7)
    lo, hi = polys.xy.min(0), polys.xy.max(0)
    pts = rng.uniform(lo - 1.0, hi + 1.0, ((RING + 1) * WARPS * TILE + 11, 2))
    check_join(og, conv, polys, idx, pts)
