"""Where one step of the points-in-polygons benchmark spends its time, piece by piece.

One step of `bench.py --workload c2` (or c4) is: free the previous index (drops the L2 persisting window and resets the
persisting lines), build the index (count kernel, host round trip for the data-dependent sizes, fill kernel), the join
(`k_pip_stream` + `k_pip_deferred`) and the per-polygon counts (`k_histogram`).  This tool runs that step on the same
inputs and prints ONE JSON line with min and median over `--reps` steps of:

* `step_ms`: CUDA events around whole steps, profiler off (what bench.py's ms_per_step measures);
* from a torch.profiler run of its own (CUDA activities): the duration of every kernel of the step, and `round_trip_us` =
  the idle gap from the end of the count kernel to the start of the fill kernel (D2H of the sizes + host synchronise +
  slab carve + cooperative launch);
* `free_us`: host time of `gpl_pip_index_free` between two stream synchronisations;
* `build_phases_us`: the `%globaltimer` stamps of both build kernels (`PipIndex.timeline()`: one thread's view), as
  durations of the phases;
* the card's name and power limit, read by nvidia-smi in the same run.

With `--split`, also `stream_split_ms`: `k_pip_stream` alone (the library's CUDA event pairs around each launch, median
over `--reps` launches after `--warmup`) on the same index for three point columns of the same size:

* `bench`: the benchmark's points (`gpl_gen_uniform_points`, stream 2);
* `no_walk`: points that never walk: uniform within +-1/4 fine cell around the centres of random fine cells whose raster
  code is 0, 1 or 2 (decoded from `PipIndex.dump("raster")`);
* `outside`: points outside the union bbox: the stream-and-write floor, no raster gather;

and `walk_ms` = bench - no_walk, `raster_ms` = no_walk - outside, and beside them `traffic_floor`: a torch op on the
benchmark's point column that reads 16 bytes and writes 4 per point, as the kernel does (see `traffic_floor`), the time
the card takes for the same traffic without any of the kernel's work.

    python tools/pip_step_breakdown.py [--workload c2|c4] [--reps 20] [--warmup 5] [--points N] [--split] [--out FILE]

Needs a CUDA device."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

# kernel name fragment -> piece
KERNELS = (("k_pip_build_count", "count"), ("k_pip_build_fill", "fill"), ("k_pip_stream", "stream"),
           ("k_pip_deferred", "deferred"), ("k_histogram", "histogram"))
# timeline stamp pairs -> phase (see PipIndex.timeline)
PHASES = (("count_S0_headers", 0, 1), ("count_S1_cells", 1, 2), ("count_S2_buckets", 2, 3), ("count_S3_plan", 3, 4),
          ("fill_T0_scans", 5, 6), ("fill_T1_prefix", 6, 7), ("fill_T2_lists", 7, 8), ("fill_T3_bucket_finish", 8, 9),
          ("fill_T4_cell_recs", 9, 10), ("fill_T4_raster", 10, 11))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                              os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0]], capture_output=True, text=True,
                             timeout=60).stdout.strip().splitlines()
        name, power, clk = (s.strip() for s in out[0].split(","))
        return {"name": name, "power_limit": power, "max_sm_clock": clk}
    except Exception as e:  # noqa: BLE001 - the numbers are still worth printing
        return {"name": "unknown", "error": str(e)}


def stat(xs, digits=2):
    xs = list(xs)
    return {"min": round(min(xs), digits), "median": round(statistics.median(xs), digits)} if xs else None


def split_columns(torch, idx, poly_xy, n, dev):
    """the `no_walk` and `outside` point columns of --split (n x 2 float64 each, on dev; seeded)"""
    st = idx.stats()
    fg = st["fine_cells_per_axis"]
    x0, y0 = (float(v) for v in poly_xy.min(dim=0).values)
    x1, y1 = (float(v) for v in poly_xy.max(dim=0).values)
    words = idx.dump("raster").view(np.uint32).reshape(fg, -1, 2)[:, :, 0]  # (fine row, word): 16 two-bit codes
    codes = (words[:, :, None] >> (2 * np.arange(16, dtype=np.uint32))) & 3
    codes = codes.reshape(fg, -1)[:, :fg]
    keep = torch.from_numpy(np.flatnonzero(codes != 3)).to(dev)
    g = torch.Generator(device=dev)
    g.manual_seed(7)
    pick = keep[torch.randint(0, keep.numel(), (n,), device=dev, generator=g)]
    fw, fh = (x1 - x0) / fg, (y1 - y0) / fg
    jit = torch.rand((n, 2), dtype=torch.float64, device=dev, generator=g) * 0.5 + 0.25  # centre +- 1/4 cell
    no_walk = torch.stack((x0 + ((pick % fg).double() + jit[:, 0]) * fw, y0 + ((pick // fg).double() + jit[:, 1]) * fh), dim=1)
    del pick, jit
    outside = torch.rand((n, 2), dtype=torch.float64, device=dev, generator=g)
    outside[:, 0] = x1 + 1.0 + outside[:, 0] * (x1 - x0)
    outside[:, 1] = y0 + outside[:, 1] * (y1 - y0)
    return no_walk.contiguous(), outside


def traffic_floor(torch, pts, stream, warmup, reps):
    """ms of a torch op that moves what k_pip_stream must move per point, 16 bytes in and 4 out: an int32 column of the
    low words of x, a strided read that still pulls every 32-byte sector of the point column.  CUDA events around the
    op; min and median over `reps`."""
    low = pts.view(torch.int32)[:, 0]
    out = torch.empty(low.shape[0], dtype=torch.int32, device=pts.device)
    for _ in range(warmup):
        out.copy_(low)
    ms = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        out.copy_(low)
        e1.record(stream)
        e1.synchronize()
        ms.append(e0.elapsed_time(e1))
    return stat(ms, 3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="c2", choices=["c2", "c4"])
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--points", type=int, default=0)
    ap.add_argument("--split", action="store_true", help="also time k_pip_stream alone on bench / no-walk / outside points")
    ap.add_argument("--out", default=None, help="also append the JSON line to this file")
    args = ap.parse_args()

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("pip_step_breakdown.py needs a CUDA device")
    from geopolars_b200 import GeometryType, synth
    from geopolars_b200 import engine as E

    if args.workload == "c2":
        n_polys, grid, cell, nvert, n = 10_000, 100, 10.0, 64, args.points or 100_000_000
    else:
        n_polys, grid, cell, nvert, n = 1_000, 32, 31.25, 64, args.points or 125_000_000
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(device=dev)
    with torch.cuda.stream(stream):
        ctx = E.Context(0, stream.cuda_stream)
        pts = torch.empty((n, 2), dtype=torch.float64, device=dev)
        E.check(ctx.lib.gpl_gen_uniform_points(ctx._h, 2, 0, n, grid * cell, pts.data_ptr()))
        xy, ro, go = synth.star_polygons(n_polys, grid, cell, nvert)
        n_pc = len(xy)
        poly_xy = torch.from_numpy(xy).to(dev)
        ring_off = torch.from_numpy(ro).to(dev)
        geom_off = torch.from_numpy(go).to(dev)
        ids = torch.empty(n, dtype=torch.int32, device=dev)
        counts = torch.zeros(n_polys, dtype=torch.int64, device=dev)
        polys = ctx.wrap_device(GeometryType.POLYGON, n_polys, n_pc, poly_xy.data_ptr(), geom_off_ptr=geom_off.data_ptr(),
                                ring_off_ptr=ring_off.data_ptr(), n_rings=n_polys, keepalive=(poly_xy, geom_off, ring_off))
        state = {"idx": None}

        def step():
            if state["idx"] is not None:
                state["idx"].free()
            state["idx"] = E.PipIndex(polys)
            state["idx"].query_device(pts.data_ptr(), n, ids.data_ptr())
            E.check(ctx.lib.gpl_join_histogram(ctx._h, ids.data_ptr(), n, counts.data_ptr(), n_polys, E.GPL_DEVICE))

        for _ in range(args.warmup):
            step()
        stream.synchronize()

        # 1. whole steps, profiler off
        step_ms = []
        for _ in range(args.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            step()
            e1.record(stream)
            e1.synchronize()
            step_ms.append(e0.elapsed_time(e1))
        # the same, back to back (as bench.py runs them: the host enqueues the next step while the GPU works)
        stream.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(args.reps):
            step()
        e1.record(stream)
        e1.synchronize()
        step_ms_back_to_back = e0.elapsed_time(e1) / args.reps

        # 2. build timeline stamps (each read synchronises: a loop of its own)
        phases = {name: [] for name, _, _ in PHASES}
        count_to_fill = []
        for _ in range(args.reps):
            step()
            t = state["idx"].timeline()
            for name, a, b in PHASES:
                phases[name].append(t[b] - t[a])
            count_to_fill.append(t[5] - t[4])
        stream.synchronize()

        # 3. free (host time between two synchronisations)
        free_us = []
        for _ in range(args.reps):
            step()
            stream.synchronize()
            t0 = time.perf_counter()
            state["idx"].free()
            stream.synchronize()
            free_us.append((time.perf_counter() - t0) * 1e6)
            state["idx"] = None

        # 4. kernels and gaps from a profiler run of its own
        for _ in range(3):
            step()
        stream.synchronize()
        from torch.profiler import ProfilerActivity, profile

        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.reps):
                step()
            stream.synchronize()
        evs = []
        for ev in prof.profiler.kineto_results.events():
            if ev.device_type() != torch.autograd.DeviceType.CUDA:
                continue
            evs.append((ev.start_ns(), ev.start_ns() + ev.duration_ns(), ev.name()))
        evs.sort()
        kern = {piece: [] for _, piece in KERNELS}
        round_trip, count_end = [], None
        for s, e, name in evs:
            piece = next((p for frag, p in KERNELS if frag in name), None)
            if piece is None:
                continue
            kern[piece].append((e - s) * 1e-3)
            if piece == "count":
                count_end = e
            elif piece == "fill" and count_end is not None:
                round_trip.append((s - count_end) * 1e-3)
                count_end = None

        # 5. --split: the stream kernel alone on one index, three point columns
        split = None
        if args.split:
            idx = state["idx"]
            no_walk, outside = split_columns(torch, idx, poly_xy, n, dev)
            split = {}
            for name, col in (("bench", pts), ("no_walk", no_walk), ("outside", outside)):
                for _ in range(args.warmup):
                    idx.query_device(col.data_ptr(), n, ids.data_ptr())
                stream.synchronize()
                ctx.kernel_timing(True)
                ms = []
                for _ in range(args.reps):
                    idx.query_device(col.data_ptr(), n, ids.data_ptr())
                    t, k = ctx.kernel_timing_read()
                    ms.append(t / k)
                ctx.kernel_timing(False)
                split[name] = stat(ms, 3)
            del no_walk, outside
            med = {k: v["median"] for k, v in split.items()}
            split["walk_ms"] = round(med["bench"] - med["no_walk"], 3)
            split["raster_ms"] = round(med["no_walk"] - med["outside"], 3)
            split["traffic_floor"] = traffic_floor(torch, pts, stream, args.warmup, args.reps)
        state["idx"].free()
        stream.synchronize()

    res = {
        "tool": "pip_step_breakdown",
        "workload": args.workload,
        "points": n,
        "polygons": n_polys,
        "reps": args.reps,
        "card": card(),
        "step_ms": stat(step_ms),
        "step_ms_back_to_back": round(step_ms_back_to_back, 4),
        "kernels_us": {k: stat(v) for k, v in kern.items()},
        "round_trip_us": stat(round_trip),
        "free_us": stat(free_us),
        "build_phases_us": {k: stat(v) for k, v in phases.items()},
        "count_end_to_fill_start_us": stat(count_to_fill),
    }
    if split is not None:
        res["stream_split_ms"] = split
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "a") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
