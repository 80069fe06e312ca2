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

    python tools/pip_step_breakdown.py [--workload c2|c4] [--reps 20] [--warmup 5] [--points N] [--out FILE]

Needs a CUDA device."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

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


def stat(xs):
    xs = list(xs)
    return {"min": round(min(xs), 2), "median": round(statistics.median(xs), 2)} if xs else None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="c2", choices=["c2", "c4"])
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--points", type=int, default=0)
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
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "a") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
