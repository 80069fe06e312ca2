"""An executable model of the index arithmetic of the batched walk in k_pip_stream<LEAN> (geopolars_b200/csrc/k_pip.cu:
walk_batch): which lane loads which record of which point in each of its three phases.

What it establishes, independently of any GPU: for any set of active points and any overflow-run lengths a list may have
(0 .. kFastMaxCount - (kFastListRecs - 1) records), every record a point's walk needs is loaded exactly once, by a lane that
attributes it to that point and to the right slot, and no other record is loaded."""
import numpy as np
import pytest

R = 6  # kFastListRecs
MAX_COUNT = 120  # kFastMaxCount
LANES = 32


def phase1(active):
    """(point, half) of every loaded cell-record half"""
    got = []
    for h in range(2):
        for lane in range(LANES):
            q = 16 * h + (lane >> 1)
            if active[q]:
                got.append((q, lane & 1))
    return got


def phase2(lists):
    """(point, slot) of every loaded list record; slot 0 is the header"""
    got = []
    for j in range(R):
        for lane in range(LANES):
            k = LANES * j + lane
            q = k // R
            if lists[q]:
                got.append((q, k - q * R))
    return got


def phase3(tail_n):
    """(point, record of its overflow run) of every loaded tail record: warp prefix sum + binary search over the run starts,
    in rounds of 4 x 32 records"""
    n = np.asarray(tail_n, dtype=np.int64)
    incl = np.cumsum(n)  # the shfl_up scan
    total = int(incl[-1])
    start = incl - n
    src = -start  # + t = record within the point's run (the kernel adds the run's table offset)
    got, rounds = [], 0
    for t0 in range(0, total, 4 * LANES):
        rounds += 1
        for u in range(4):
            for lane in range(LANES):
                t = t0 + LANES * u + lane
                q = 0
                for step in (16, 8, 4, 2, 1):
                    if start[q + step] <= t:
                        q += step
                if t < total:
                    got.append((q, int(src[q] + t)))
    return got, rounds, total


def expect(mask, per_point):
    return sorted((q, s) for q in range(LANES) if mask[q] for s in range(per_point(q)))


@pytest.mark.parametrize("seed", range(40))
def test_every_record_loaded_once_by_its_point(seed):
    rng = np.random.default_rng(seed)
    active = rng.random(LANES) < rng.choice([0.3, 0.9, 1.0])
    lists = active & (rng.random(LANES) < rng.choice([0.5, 1.0]))
    count = rng.integers(0, MAX_COUNT + 1, LANES)
    if seed % 4 == 0:
        count[:] = MAX_COUNT  # every point takes the longest list
    tail_n = np.where(lists, np.maximum(count - (R - 1), 0), 0)

    got1 = phase1(active)
    assert sorted(got1) == expect(active, lambda q: 2)
    got2 = phase2(lists)
    assert sorted(got2) == expect(lists, lambda q: R)
    got3, rounds, total = phase3(tail_n)
    assert sorted(got3) == expect(tail_n > 0, lambda q: int(tail_n[q]))
    assert total == tail_n.sum() and rounds == -(-total // (4 * LANES))


def test_longest_batch_and_empty_runs():
    """32 runs of the longest length (29 rounds), and runs of length 0 between non-empty ones (equal starts)"""
    full = np.full(LANES, MAX_COUNT - (R - 1))
    got, rounds, total = phase3(full)
    assert total == LANES * (MAX_COUNT - (R - 1)) and rounds == 29
    assert sorted(got) == expect(full > 0, lambda q: int(full[q]))
    sparse = np.zeros(LANES, dtype=np.int64)
    sparse[[0, 5, 6, 31]] = [1, 115, 2, 3]
    got, _, _ = phase3(sparse)
    assert sorted(got) == expect(sparse > 0, lambda q: int(sparse[q]))
