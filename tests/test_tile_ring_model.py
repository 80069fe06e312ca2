"""An executable model of the output path of k_pip_stream (geopolars_b200/csrc/k_pip.cu): the per-warp ring of kRing tile
slots in shared memory and the FIFO queue of walked points.

It restates one warp's loop: tile j goes to slot j & (kRing - 1), its code-3 points are appended to a circular queue of
kQueueCap entries (k-major, lane-minor: ascending row in the tile), the warp walks its 32 oldest entries while 32 are
queued, then whatever is left of the tile whose slot the next tile takes (a partial batch if fewer than 32 are queued),
and everything after its last tile, and a slot is stored as one whole tile when the next tile takes it or at the end.

What it establishes, independently of any GPU, for random walker patterns (every point of a tile walked, none, sparse,
clustered): every tile is stored exactly once, after the last walk of any of its points; every walked point is walked
exactly once and its result lands in the slot that holds its tile; no slot is taken while a point of its tile is still
queued; the queue never holds more than kQueueCap entries; and the index the kernel appends to the deferred list
(ring_tile[at / kTilePts] * kTilePts + at % kTilePts) is the point's row."""
import numpy as np
import pytest

K = 4  # kRing
TILE = 128  # kTilePts
CAP = TILE + 32  # kQueueCap
LANES = 32


def run_warp(walk_masks, t0, n_warps, n_pts):
    """one warp over tiles t0, t0 + n_warps, ... (walk_masks[j]: which of tile j's 128 rows have raster code 3).
    Returns the event log: ("walk", row, slot, batch size) per walked point, ("store", tile) per stored tile."""
    q = [None] * CAP  # entry: at = slot * TILE + row in the tile
    qh = qn = 0
    ring_tile = [None] * K
    pending = [0] * K  # the model's own bookkeeping (the kernel has none): queued points of the tile in each slot
    log = []

    def walk_oldest(n):
        nonlocal qh, qn
        assert 1 <= n <= LANES and n <= qn
        for lane in range(n):
            e = qh + lane if qh + lane < CAP else qh + lane - CAP
            at = q[e]
            q[e] = None
            s = at // TILE
            pending[s] -= 1
            log.append(("walk", ring_tile[s] * TILE + at % TILE, s, n))
        qh = qh + n if qh + n < CAP else qh + n - CAP
        qn -= n

    def flush(s):
        assert pending[s] == 0, "a tile is stored while points of it are queued"
        log.append(("store", ring_tile[s]))

    n_tiles = -(-n_pts // TILE)
    j = 0
    tile = t0
    while tile < n_tiles:
        s = j & (K - 1)
        assert pending[s] == 0, "a slot is taken while points of its tile are queued"
        ring_tile[s] = tile
        rows = [r for r in range(TILE) if walk_masks[j][r] and tile * TILE + r < n_pts]
        for k in range(TILE // LANES):  # stage 4: one ballot per k, lanes in order
            for lane in range(LANES):
                r = lane + LANES * k
                if r in rows:
                    pos = qh + qn
                    pos = pos - CAP if pos >= CAP else pos
                    assert q[pos] is None, "the queue overwrote a waiting entry"
                    q[pos] = s * TILE + r
                    qn += 1
                    pending[s] += 1
        assert qn <= CAP
        s_next = (j + 1) & (K - 1)
        last = tile + n_warps >= n_tiles
        while qn >= 32 or (qn > 0 and (last or q[qh] // TILE == s_next)):
            walk_oldest(min(qn, 32))
        if j + 1 >= K:
            flush(s_next)
        tile += n_warps
        j += 1
    for d in range(1, K):
        if d <= j:
            flush((j - d) & (K - 1))
    assert qn == 0
    return log


def check(walk_masks, t0, n_warps, n_pts):
    log = run_warp(walk_masks, t0, n_warps, n_pts)
    n_tiles = -(-n_pts // TILE)
    tiles = list(range(t0, n_tiles, n_warps))
    stored = [e[1] for e in log if e[0] == "store"]
    assert sorted(stored) == tiles  # every tile exactly once
    want = {t * TILE + r for j, t in enumerate(tiles) for r in range(TILE) if walk_masks[j][r] and t * TILE + r < n_pts}
    walked = [e[1] for e in log if e[0] == "walk"]
    assert len(walked) == len(set(walked)) and set(walked) == want  # every walker exactly once, at its row
    store_at = {e[1]: i for i, e in enumerate(log) if e[0] == "store"}
    for i, e in enumerate(log):
        if e[0] == "walk":
            assert i < store_at[e[1] // TILE]  # stored after its tile's last walker
    # the oldest entries go first: walks follow the rows' order in the warp's stream
    assert walked == sorted(walked)
    return log


def masks(rng, n, kind):
    if kind == "all":
        return np.ones((n, TILE), bool)
    if kind == "none":
        return np.zeros((n, TILE), bool)
    if kind == "clustered":  # runs of tiles that walk everything, nothing, or a few
        out = np.zeros((n, TILE), bool)
        for j in range(n):
            out[j] = rng.random(TILE) < rng.choice([0.0, 0.02, 0.06, 1.0])
        return out
    return rng.random((n, TILE)) < kind


@pytest.mark.parametrize("kind", ["all", "none", "clustered", 0.01, 0.06, 0.228, 0.5, 0.9])
@pytest.mark.parametrize("seed", range(6))
def test_ring_and_fifo(kind, seed):
    rng = np.random.default_rng(seed)
    n_warps = int(rng.integers(1, 40))
    t0 = int(rng.integers(0, n_warps))
    n_tiles = t0 + n_warps * int(rng.integers(0, 30)) + int(rng.integers(0, n_warps + 1))
    n_pts = max(1, n_tiles * TILE - int(rng.integers(0, TILE)))
    n_mine = len(range(t0, -(-n_pts // TILE), n_warps))
    check(masks(rng, n_mine, kind), t0, n_warps, n_pts)


@pytest.mark.parametrize("n_pts", [1, 31, 127, 128, 129, 1000, K * TILE, K * TILE + 1, 3 * K * TILE - 5])
def test_sizes_one_warp(n_pts):
    rng = np.random.default_rng(n_pts)
    n_mine = -(-n_pts // TILE)
    check(rng.random((n_mine, TILE)) < 0.3, 0, 1, n_pts)


def test_walker_resolved_ring_tiles_later():
    """sparse walkers (fewer than 32 in any kRing - 1 consecutive tiles) wait in the queue until a slot is needed: tile 0's
    walker is walked, with the two queued after it, in one partial batch just before tile kRing takes slot 0"""
    m = np.zeros((12, TILE), bool)
    m[0, 5] = m[1, 7] = m[2, 9] = True
    log = check(m, 0, 1, 12 * TILE)
    walks = [e for e in log if e[0] == "walk"]
    assert [(w[1], w[3]) for w in walks] == [(5, 3), (TILE + 7, 3), (2 * TILE + 9, 3)]
    # the first walk comes after tile kRing - 1 was queued: no tile was stored before it
    first_walk = next(i for i, e in enumerate(log) if e[0] == "walk")
    assert not any(e[0] == "store" for e in log[:first_walk])


def test_full_tiles_force_nothing():
    """with every point walked, each tile leaves as 4 full batches and the queue never holds more than one tile"""
    log = check(np.ones((10, TILE), bool), 0, 1, 10 * TILE)
    assert {e[3] for e in log if e[0] == "walk"} == {32}
