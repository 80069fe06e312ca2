#!/usr/bin/env python
"""Kernel-resident timings of the other §8 rows at BASELINE config sizes (3 and 5), with the HBM roofline
fraction for the coordinate bytes read, and of the nearest join (100 M points against config 2's polygons, 1 M
reference points and 1 M walk linestrings).  Not the flagship bench (that is bench.py, config 2); config 5 runs at
4 M polygons so that its input and output columns fit one 80 GB H100.

  python tools/bench_ops.py [--scale 1.0] [--only all|ops|nearest|nearest_geom|dwithin|geo|overlay|geodesic|valid|boolean|relate|dissolve|clip|overlay_modes] [--out ops_roofline.json]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from geopolars_b200 import GeometryType  # noqa: E402
from geopolars_b200 import engine as E  # noqa: E402


def timed(stream, fn, reps=5, warm=2):
    for _ in range(warm):
        fn()
    stream.synchronize()
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        fn()
        e1.record(stream)
        stream.synchronize()
        ts.append(e0.elapsed_time(e1))
    return min(ts), sum(ts) / len(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=float, default=1.0, help="fraction of the BASELINE sizes")
    ap.add_argument("--out", default="ops_roofline.json")
    ap.add_argument("--only", choices=("all", "ops", "nearest", "nearest_geom", "dwithin", "geo", "overlay", "geodesic", "valid", "boolean", "relate", "dissolve", "clip", "overlay_modes"), default="all",
                    help="run only the §8 rows, only the point nearest join, only the geometry nearest join, only the "
                         "distance-within join, only the great-circle joins, only the intersection area and overlay join or "
                         "only the geodesic area and perimeter (1 M stars, 10 M parcels, naturalearth_lowres to 1 M rows), or only "
                         "the boolean geometry ops and the geometry overlay join, or only the DE-9IM relate, predicates and "
                         "predicate join, or only dissolve / union_all, or only the line clip, intersection length and their joins, or "
                         "only the symmetric difference and the five overlay modes; "
                         "'all' runs every arm")
    args = ap.parse_args()
    peak = 3350.0  # H100 SXM data sheet, replaced by a measured value when MEASURED_PEAKS.json exists
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        peak = float(json.load(open(p)).get("hbm_gbs", peak))
    dev = torch.device("cuda", 0)
    st = torch.cuda.Stream()
    res = {"peak_hbm_GBps": peak, "rows": []}

    def row(name, units, unit_name, bytes_read, bytes_written, t_min, t_avg):
        r = {"op": name, "units": units, "unit": unit_name, "ms_min": t_min, "ms_avg": t_avg, "units_per_s": units / (t_avg * 1e-3),
             "read_GBps": bytes_read / (t_avg * 1e-3) / 1e9, "read_write_GBps": (bytes_read + bytes_written) / (t_avg * 1e-3) / 1e9,
             "frac_read": bytes_read / (t_avg * 1e-3) / 1e9 / peak, "frac_read_write": (bytes_read + bytes_written) / (t_avg * 1e-3) / 1e9 / peak}
        res["rows"].append(r)
        print(json.dumps(r), flush=True)

    res["card"] = torch.cuda.get_device_name(0)
    try:  # read-only query: the power limit is part of every number below
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                           timeout=30)
        res["power_limit"] = q.stdout.strip().split(",")[-1].strip() if q.returncode == 0 else "unknown"
    except (OSError, subprocess.SubprocessError):
        res["power_limit"] = "unknown"
    print(json.dumps({"card": res["card"], "power_limit": res["power_limit"]}), flush=True)
    with torch.cuda.stream(st):
        ctx = E.Context(0, st.cuda_stream)
        lib = ctx.lib
        if args.only in ("all", "nearest"):
            nearest_rows(args, ctx, dev, st, res)
        if args.only in ("all", "nearest_geom"):
            nearest_geom_rows(args, ctx, dev, st, res)
        if args.only in ("all", "dwithin"):
            dwithin_rows(args, ctx, dev, st, res)
        if args.only in ("all", "geo"):
            geo_rows(args, ctx, dev, st, res)
        if args.only in ("all", "overlay"):
            overlay_rows(args, ctx, dev, st, res)
        if args.only in ("all", "boolean"):
            boolean_rows(args, ctx, dev, st, res)
        if args.only in ("all", "relate"):
            relate_rows(args, ctx, dev, st, res)
        if args.only in ("all", "dissolve"):
            dissolve_rows(args, ctx, dev, st, res)
        if args.only in ("all", "clip"):
            clip_rows(args, ctx, dev, st, res)
        if args.only in ("all", "overlay_modes"):
            overlay_modes_rows(args, ctx, dev, st, res)
        if args.only in ("all", "geodesic"):
            geodesic_rows(args, ctx, dev, st, res)
        if args.only in ("all", "valid"):
            valid_rows(args, ctx, dev, st, res)
        if args.only in ("nearest", "nearest_geom", "dwithin", "geo", "overlay", "geodesic", "valid", "boolean", "relate", "dissolve", "clip", "overlay_modes"):
            ctx.synchronize()
            _write(args, res)
            return
        # ---- config 5: G polygons x 257 coords: affine, area, centroid, convex_hull ----------------------
        G, NV = int(4_000_000 * args.scale), 256
        nc = G * (NV + 1)
        xy = torch.empty((nc, 2), dtype=torch.float64, device=dev)
        ro = torch.empty(G + 1, dtype=torch.int64, device=dev)
        go = torch.empty(G + 1, dtype=torch.int64, device=dev)
        E.check(lib.gpl_gen_blob_polygons(ctx._h, 5, 0, G, NV, xy.data_ptr(), ro.data_ptr(), go.data_ptr()))
        polys = ctx.wrap_device(GeometryType.POLYGON, G, nc, xy.data_ptr(), geom_off_ptr=go.data_ptr(), ring_off_ptr=ro.data_ptr(),
                                n_rings=G, keepalive=(xy, ro, go))
        out_f = torch.empty(G, dtype=torch.float64, device=dev)
        keep = {}

        def affine():
            keep["a"] = E.affine_transform(polys, (0.8, -0.6, 10.0, 0.6, 0.8, -5.0))

        t = timed(st, affine)
        keep.clear()
        row("affine_transform (config 5)", G, "polygons", nc * 16, nc * 16, *t)
        t = timed(st, lambda: E.check(lib.gpl_area(ctx._h, polys._h, C.c_void_p(out_f.data_ptr()), E.GPL_DEVICE)))
        row("area (config 5)", G, "polygons", nc * 16 + (G + 1) * 16, G * 8, *t)

        def cen():
            keep["c"] = E.centroid(polys)

        t = timed(st, cen)
        keep.clear()
        row("centroid (config 5)", G, "polygons", nc * 16 + (G + 1) * 16, G * 17, *t)

        def hull():
            keep["h"] = E.convex_hull(polys)

        t = timed(st, hull, reps=3, warm=1)
        hv = keep["h"].view()
        row("convex_hull (config 5)", G, "polygons", nc * 16, hv.n_coords * 16, *t)
        res["hull_mean_vertices"] = hv.n_coords / G
        keep.clear()
        # ---- WKB codec on the same polygons (§8f rank 1): encode to device WKB, decode back ---------------
        ctx.trim()  # hand the cached affine / hull blocks back: the WKB image of config 5 is another 41 GB
        wkb_bytes = G * (13 + 16 * (NV + 1))
        wb = torch.empty(wkb_bytes + 64, dtype=torch.uint8, device=dev)
        wo = torch.empty(G + 1, dtype=torch.int64, device=dev)
        t = timed(st, lambda: polys.encode_wkb(64, device_out=(wo.data_ptr(), wb.data_ptr(), wb.numel())), reps=3, warm=1)
        row("WKB encode, polygons x 257 coords (device to device)", G, "polygons", nc * 16, wkb_bytes, *t)

        def dec():
            keep["d"] = ctx.decode_wkb(wb.data_ptr(), wo.data_ptr(), None, n=G, offset_width=64, device=True)

        t = timed(st, dec, reps=3, warm=1)
        dv = keep["d"].view()
        assert dv.n_coords == nc and dv.n_rings == G
        out_g = torch.empty(G, dtype=torch.float64, device=dev)  # same areas <=> same rings (bit-exact kernel, same order)
        E.check(lib.gpl_area(ctx._h, keep["d"]._h, C.c_void_p(out_g.data_ptr()), E.GPL_DEVICE))
        st.synchronize()
        assert torch.equal(out_g, out_f), "WKB round trip changed the polygons"
        del out_g
        row("WKB decode, polygons x 257 coords (device to device)", G, "polygons", wkb_bytes, nc * 16, *t)
        keep.clear()
        del wb, wo
        # Point columns: 21-byte rows (what data/cities.arrow and the reference's point datasets hold)
        NP = int(100_000_000 * args.scale)
        pxy = torch.empty((NP, 2), dtype=torch.float64, device=dev)
        E.check(lib.gpl_gen_uniform_points(ctx._h, 2, 0, NP, 1000.0, pxy.data_ptr()))
        pts = ctx.wrap_device(GeometryType.POINT, NP, NP, pxy.data_ptr(), keepalive=(pxy,))
        wb = torch.empty(NP * 21 + 64, dtype=torch.uint8, device=dev)
        wo = torch.empty(NP + 1, dtype=torch.int32, device=dev)
        t = timed(st, lambda: pts.encode_wkb(32, device_out=(wo.data_ptr(), wb.data_ptr(), wb.numel())), reps=3, warm=1)
        row("WKB encode, points (device to device)", NP, "points", NP * 16, NP * 21 + NP * 4, *t)

        def decp():
            keep["d"] = ctx.decode_wkb(wb.data_ptr(), wo.data_ptr(), None, n=NP, offset_width=32, device=True)

        t = timed(st, decp, reps=3, warm=1)
        back = torch.empty((NP, 2), dtype=torch.float64, device=dev)
        E.check(lib.gpl_array_copy_out(ctx._h, keep["d"]._h, C.c_void_p(back.data_ptr()), None, None, None, None, E.GPL_DEVICE))
        st.synchronize()
        assert torch.equal(back, pxy), "WKB round trip changed the points"
        row("WKB decode, points (device to device)", NP, "points", NP * 21 + NP * 4, NP * 16, *t)
        keep.clear()
        del back, wb, wo, pts, pxy
        del polys, xy, ro, go, out_f
        torch.cuda.empty_cache()
        # ---- config 3: N linestring pairs, K = 16 -----------------------------------------------------------
        N, K = int(50_000_000 * args.scale), 16
        axy = torch.empty((N * K, 2), dtype=torch.float64, device=dev)
        bxy = torch.empty((N * K, 2), dtype=torch.float64, device=dev)
        aoff = torch.empty(N + 1, dtype=torch.int64, device=dev)
        boff = torch.empty(N + 1, dtype=torch.int64, device=dev)
        E.check(lib.gpl_gen_walk_linestrings(ctx._h, 3, -1, 0, N, K, axy.data_ptr(), aoff.data_ptr()))
        E.check(lib.gpl_gen_walk_linestrings(ctx._h, 4, 3, 0, N, K, bxy.data_ptr(), boff.data_ptr()))
        A = ctx.wrap_device(GeometryType.LINESTRING, N, N * K, axy.data_ptr(), geom_off_ptr=aoff.data_ptr(), keepalive=(axy, aoff))
        B = ctx.wrap_device(GeometryType.LINESTRING, N, N * K, bxy.data_ptr(), geom_off_ptr=boff.data_ptr(), keepalive=(bxy, boff))
        bm = torch.empty((N + 7) // 8, dtype=torch.uint8, device=dev)
        dist = torch.empty(N, dtype=torch.float64, device=dev)
        t = timed(st, lambda: E.check(lib.gpl_intersects(ctx._h, A._h, B._h, C.c_void_p(bm.data_ptr()), E.GPL_DEVICE)), reps=3, warm=1)
        row("intersects LineString pairs (config 3)", N, "pairs", 2 * N * K * 16 + 2 * (N + 1) * 8, N // 8, *t)
        t = timed(st, lambda: E.check(lib.gpl_distance(ctx._h, A._h, B._h, C.c_void_p(dist.data_ptr()), None, E.GPL_DEVICE)), reps=3, warm=1)
        row("distance LineString pairs (config 3, includes the intersects test)", N, "pairs", 2 * N * K * 16 + 2 * (N + 1) * 8, N * 8, *t)
        res["intersect_fraction"] = float((dist == 0).float().mean().item())
    _write(args, res)


def _write(args, res):
    if os.path.dirname(args.out):
        os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)
    print("wrote", args.out)


def nearest_rows(args, ctx, dev, st, res):
    """nearest join, kernel resident: build ms, query ms, G points/s and exact evaluations per point"""
    from geopolars_b200 import synth

    lib = ctx.lib
    NP = int(100_000_000 * args.scale)
    pts = torch.empty((NP, 2), dtype=torch.float64, device=dev)
    E.check(lib.gpl_gen_uniform_points(ctx._h, 2, 0, NP, 1000.0, pts.data_ptr()))
    nid = torch.empty(NP, dtype=torch.int32, device=dev)
    dist = torch.empty(NP, dtype=torch.float64, device=dev)
    tied = torch.empty(NP, dtype=torch.int32, device=dev)

    def run(name, rhs, n_rhs):
        tb = timed(st, lambda: E.NearestIndex(rhs).free(), reps=3, warm=1)
        idx = E.NearestIndex(rhs)
        t = timed(st, lambda: idx.query_device(pts.data_ptr(), NP, None, nid.data_ptr(), dist.data_ptr(), tied.data_ptr()), reps=3, warm=1)
        s = idx.stats()
        r = {"op": f"nearest join: {NP} uniform points x {name}", "points": NP, "rhs_rows": n_rhs, "build_ms_min": tb[0], "query_ms_min": t[0],
             "query_ms_avg": t[1], "Gpoints_per_s": NP / (t[1] * 1e-3) / 1e9, "evals_per_point": s["evaluations"] / NP,
             "overflow_points": s["overflow_points"], "grid_cells_per_axis": s["grid_cells_per_axis"], "index_bytes": s["bytes"],
             "card": res["card"], "power_limit": res["power_limit"]}
        idx.free()
        res["rows"].append(r)
        print(json.dumps(r), flush=True)

    # config 2's 10 k 64-vertex star polygons on a 100 x 100 lattice of 10-unit cells (the points' 1000 x 1000 square)
    m, nv = 10_000, 64
    xy, ro, go = synth.star_polygons(m, 100, 10.0, nv)
    pxy, pro, pgo = (torch.from_numpy(a).to(dev) for a in (xy, ro, go))
    polys = ctx.wrap_device(GeometryType.POLYGON, m, m * (nv + 1), pxy.data_ptr(), geom_off_ptr=pgo.data_ptr(), ring_off_ptr=pro.data_ptr(),
                            n_rings=m, keepalive=(pxy, pro, pgo))
    run("config 2's 10 k 64-vertex polygons", polys, m)
    # CPU arm: the independent reference of the tests (its own ring search in Python, the C oracle's distances), one core
    import time

    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import nearest_reference as nr
    from oracle import oracle as og

    k = 2000
    a = og.OGArray(og.POLYGON, xy, geom_off=go, ring_off=ro)
    host_pts = pts[:k].cpu().numpy()
    t0 = time.perf_counter()
    nr.nearest_join(a, host_pts, use_grid=True)
    dt = time.perf_counter() - t0
    r = {"op": f"nearest join CPU arm: the test reference (Python ring search + C oracle distances, one core), {k}-point prefix x "
               "config 2's polygons", "points": k, "seconds": dt, "points_per_s": k / dt}
    res["rows"].append(r)
    print(json.dumps(r), flush=True)
    # 1 M uniform reference points in the same square
    R = int(1_000_000 * max(args.scale, 0.01))
    rxy = torch.empty((R, 2), dtype=torch.float64, device=dev)
    E.check(lib.gpl_gen_uniform_points(ctx._h, 7, 0, R, 1000.0, rxy.data_ptr()))
    refs = ctx.wrap_device(GeometryType.POINT, R, R, rxy.data_ptr(), keepalive=(rxy,))
    run(f"{R} uniform reference points", refs, R)
    # 1 M 16-vertex random-walk linestrings (config 3's generator)
    K = 16
    lxy = torch.empty((R * K, 2), dtype=torch.float64, device=dev)
    loff = torch.empty(R + 1, dtype=torch.int64, device=dev)
    E.check(lib.gpl_gen_walk_linestrings(ctx._h, 3, -1, 0, R, K, lxy.data_ptr(), loff.data_ptr()))
    lines = ctx.wrap_device(GeometryType.LINESTRING, R, R * K, lxy.data_ptr(), geom_off_ptr=loff.data_ptr(), keepalive=(lxy, loff))
    ctx.synchronize()
    res["walk_linestring_extent"] = [float(v) for v in torch.cat([lxy.min(0).values, lxy.max(0).values]).cpu()]
    run(f"{R} {K}-vertex walk linestrings", lines, R)
    del pts, nid, dist, tied
    torch.cuda.empty_cache()


def nearest_geom_rows(args, ctx, dev, st, res):
    """nearest join with a non-Point left side (DESIGN.md §4.13): build ms, query ms (dense outputs to the host), left
    rows/s and exact evaluations per left row"""
    import time

    from geopolars_b200 import synth

    lib = ctx.lib

    def run(name, lhs, n_lhs, rhs, n_rhs):
        tb = timed(st, lambda: E.NearestIndex(rhs).free(), reps=3, warm=1)
        idx = E.NearestIndex(rhs)
        t = timed(st, lambda: idx.query_geom(lhs), reps=3, warm=1)
        s = idx.stats()
        r = {"op": f"nearest join (geometry left side): {name}", "left_rows": n_lhs, "rhs_rows": n_rhs, "build_ms_min": tb[0],
             "query_ms_min": t[0], "query_ms_avg": t[1], "left_rows_per_s": n_lhs / (t[1] * 1e-3), "evals_per_left_row": s["evaluations"] / n_lhs,
             "grid_cells_per_axis": s["grid_cells_per_axis"], "card": res["card"], "power_limit": res["power_limit"]}
        idx.free()
        res["rows"].append(r)
        print(json.dumps(r), flush=True)

    m, nv = 10_000, 64
    xy, ro, go = synth.star_polygons(m, 100, 10.0, nv)
    pxy, pro, pgo = (torch.from_numpy(a).to(dev) for a in (xy, ro, go))
    polys = ctx.wrap_device(GeometryType.POLYGON, m, m * (nv + 1), pxy.data_ptr(), geom_off_ptr=pgo.data_ptr(), ring_off_ptr=pro.data_ptr(),
                            n_rings=m, keepalive=(pxy, pro, pgo))
    R, K = int(1_000_000 * max(args.scale, 0.01)), 16
    lxy = torch.empty((R * K, 2), dtype=torch.float64, device=dev)
    loff = torch.empty(R + 1, dtype=torch.int64, device=dev)
    E.check(lib.gpl_gen_walk_linestrings(ctx._h, 3, -1, 0, R, K, lxy.data_ptr(), loff.data_ptr()))
    lines = ctx.wrap_device(GeometryType.LINESTRING, R, R * K, lxy.data_ptr(), geom_off_ptr=loff.data_ptr(), keepalive=(lxy, loff))
    ctx.synchronize()
    run(f"{R} {K}-vertex walk linestrings x config 2's 10 k 64-vertex polygons", lines, R, polys, m)
    rxy = torch.empty((R, 2), dtype=torch.float64, device=dev)
    E.check(lib.gpl_gen_uniform_points(ctx._h, 7, 0, R, 1000.0, rxy.data_ptr()))
    refs = ctx.wrap_device(GeometryType.POINT, R, R, rxy.data_ptr(), keepalive=(rxy,))
    ctx.synchronize()
    run(f"config 2's 10 k 64-vertex polygons x {R} uniform points", polys, m, refs, R)
    # CPU arm: the independent reference of the tests (best-first search in Python, the C oracle's distances), one core
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import nearest_geom_reference as ngr
    from oracle import oracle as og

    k = 200
    a = og.OGArray(og.POLYGON, xy, geom_off=go, ring_off=ro)
    lx, lo = lxy[:k * K].cpu().numpy(), loff[:k + 1].cpu().numpy()
    left = og.OGArray(og.LINESTRING, lx, geom_off=lo)
    t0 = time.perf_counter()
    ngr.nearest_join_geom(left, a, use_pruning=True)
    dt = time.perf_counter() - t0
    r = {"op": f"nearest join (geometry left side) CPU arm: the test reference (Python best-first search + C oracle distances, one core), "
               f"{k}-row prefix of the walk linestrings x config 2's polygons", "left_rows": k, "seconds": dt, "left_rows_per_s": k / dt}
    res["rows"].append(r)
    print(json.dumps(r), flush=True)
    del lxy, loff, rxy
    torch.cuda.empty_cache()


def dwithin_rows(args, ctx, dev, st, res):
    """distance-within join (DESIGN.md §4.14), kernel resident: build ms, count-pass ms (dense counts in HBM), pair-list ms
    (device-resident gpl_pairs with distances, freed after each call), left rows/s, pairs/s, exact evaluations per left row of
    the last pass and pairs returned; plus a cKDTree CPU arm for workload 1"""
    import time

    from geopolars_b200 import synth

    lib = ctx.lib

    def run(name, lhs, n_lhs, rhs, n_rhs, D):
        tb = timed(st, lambda: E.NearestIndex(rhs).free(), reps=3, warm=1)
        idx = E.NearestIndex(rhs)
        cnt = torch.empty(max(n_lhs, 1), dtype=torch.int32, device=dev)
        tc = timed(st, lambda: E.check(lib.gpl_dwithin_count(ctx._h, idx._h, lhs._h, D, C.c_void_p(cnt.data_ptr()), E.GPL_DEVICE)), reps=3, warm=1)
        evals_count = idx.stats()["evaluations"]
        n_pairs = [0]

        def pairs():
            h = C.c_void_p()
            E.check(lib.gpl_dwithin_join_pairs(ctx._h, idx._h, lhs._h, D, 1, C.byref(h)))
            n_pairs[0] = int(lib.gpl_pairs_count(h))
            lib.gpl_pairs_free(h)

        tp = timed(st, pairs, reps=3, warm=1)
        s = idx.stats()
        r = {"op": f"dwithin join: {name}, D = {D}", "left_rows": n_lhs, "rhs_rows": n_rhs, "distance": D, "build_ms_min": tb[0],
             "count_ms_min": tc[0], "count_ms_avg": tc[1], "pairs_ms_min": tp[0], "pairs_ms_avg": tp[1],
             "count_left_rows_per_s": n_lhs / (tc[1] * 1e-3), "pairs_left_rows_per_s": n_lhs / (tp[1] * 1e-3),
             "pairs_per_s": n_pairs[0] / (tp[1] * 1e-3), "evals_per_left_row": evals_count / n_lhs,
             "evals_per_left_row_write_pass": s["evaluations"] / n_lhs, "pairs": n_pairs[0], "total_count": int(cnt[:n_lhs].sum().item()),
             "grid_cells_per_axis": s["grid_cells_per_axis"], "card": res["card"], "power_limit": res["power_limit"]}
        idx.free()
        res["rows"].append(r)
        print(json.dumps(r), flush=True)

    NP, NR = int(10_000_000 * max(args.scale, 0.01)), int(1_000_000 * max(args.scale, 0.01))
    lp = torch.empty((NP, 2), dtype=torch.float64, device=dev)
    rp = torch.empty((NR, 2), dtype=torch.float64, device=dev)
    E.check(lib.gpl_gen_uniform_points(ctx._h, 1, 0, NP, 1000.0, lp.data_ptr()))
    E.check(lib.gpl_gen_uniform_points(ctx._h, 2, 0, NR, 1000.0, rp.data_ptr()))
    left = ctx.wrap_device(GeometryType.POINT, NP, NP, lp.data_ptr(), keepalive=(lp,))
    refs = ctx.wrap_device(GeometryType.POINT, NR, NR, rp.data_ptr(), keepalive=(rp,))
    ctx.synchronize()
    # 1: 10 M x 1 M uniform points, D = 1 (about pi matches per point)
    run(f"{NP} uniform points x {NR} uniform points", left, NP, refs, NR, 1.0)
    # 2: 10 M uniform points x config 2's 10 k 64-vertex polygons, D = 0.5
    m, nv = 10_000, 64
    xy, ro, go = synth.star_polygons(m, 100, 10.0, nv)
    pxy, pro, pgo = (torch.from_numpy(a).to(dev) for a in (xy, ro, go))
    polys = ctx.wrap_device(GeometryType.POLYGON, m, m * (nv + 1), pxy.data_ptr(), geom_off_ptr=pgo.data_ptr(), ring_off_ptr=pro.data_ptr(),
                            n_rings=m, keepalive=(pxy, pro, pgo))
    run(f"{NP} uniform points x config 2's 10 k 64-vertex polygons", left, NP, polys, m, 0.5)
    # 3: 1 M 16-vertex walk linestrings x config 2's polygons, D = 1
    K = 16
    lxy = torch.empty((NR * K, 2), dtype=torch.float64, device=dev)
    loff = torch.empty(NR + 1, dtype=torch.int64, device=dev)
    E.check(lib.gpl_gen_walk_linestrings(ctx._h, 3, -1, 0, NR, K, lxy.data_ptr(), loff.data_ptr()))
    lines = ctx.wrap_device(GeometryType.LINESTRING, NR, NR * K, lxy.data_ptr(), geom_off_ptr=loff.data_ptr(), keepalive=(lxy, loff))
    ctx.synchronize()
    run(f"{NR} {K}-vertex walk linestrings x config 2's polygons", lines, NR, polys, m, 1.0)
    del lxy, loff, lines
    # 4: workload 1 with the left side as one-member MultiPoint rows: the warp-per-row kernel on the same pairs
    moff = torch.arange(NP + 1, dtype=torch.int64, device=dev)
    mleft = ctx.wrap_device(GeometryType.MULTIPOINT, NP, NP, lp.data_ptr(), geom_off_ptr=moff.data_ptr(), keepalive=(lp, moff))
    ctx.synchronize()
    run(f"{NP} one-member MultiPoint rows x {NR} uniform points", mleft, NP, refs, NR, 1.0)
    # CPU arm of workload 1: scipy's cKDTree.query_ball_point on every core of this host, on a prefix of the left points
    from scipy.spatial import cKDTree

    k = min(NP, 2_000_000)
    L, R = lp[:k].cpu().numpy(), rp.cpu().numpy()
    t0 = time.perf_counter()
    tree = cKDTree(R)
    t1 = time.perf_counter()
    nb = tree.query_ball_point(L, 1.0, workers=-1, return_length=True)
    t2 = time.perf_counter()
    r = {"op": f"dwithin join CPU arm: scipy cKDTree.query_ball_point(workers=-1, return_length=True), {k}-point prefix of workload 1",
         "left_rows": k, "nproc": os.cpu_count(), "build_s": t1 - t0, "query_s": t2 - t1, "left_rows_per_s": k / (t2 - t1),
         "pairs": int(nb.sum()), "pairs_per_s": int(nb.sum()) / (t2 - t1)}
    res["rows"].append(r)
    print(json.dumps(r), flush=True)
    del lp, rp, pxy, pro, pgo, moff
    torch.cuda.empty_cache()


def overlay_rows(args, ctx, dev, st, res):
    """intersection area (DESIGN.md §4.16), kernel resident: row-wise on 1 M pairs of config 2's 65-coordinate stars against
    the same stars shifted by (3, 2), and the overlay join of config 2's 10 000 stars against a 1000 x 1000 grid of unit
    squares (candidate stage + exact intersects + area, host synchronisations included).  ms, pairs/s and edge pairs/s
    (the (edge of A, edge of B) pairs of the evaluated row pairs, each examined once per pass): the kernel is FP64 bound."""
    import numpy as np

    from geopolars_b200 import synth

    lib = ctx.lib

    def rec(name, units, unit_name, edge_pairs, t):
        r = {"op": name, "units": units, "unit": unit_name, "ms_min": t[0], "ms_avg": t[1], "units_per_s": units / (t[1] * 1e-3),
             "edge_pairs": edge_pairs, "edge_pairs_per_s": edge_pairs / (t[1] * 1e-3), "card": res["card"], "power_limit": res["power_limit"]}
        res["rows"].append(r)
        print(json.dumps(r), flush=True)

    def upload(xy, ring_off, geom_off):
        t = [torch.from_numpy(np.ascontiguousarray(v)).to(dev) for v in (xy, ring_off, geom_off)]
        n = len(geom_off) - 1
        return ctx.wrap_device(GeometryType.POLYGON, n, len(xy), t[0].data_ptr(), geom_off_ptr=t[2].data_ptr(), ring_off_ptr=t[1].data_ptr(),
                               n_rings=len(ring_off) - 1, keepalive=tuple(t))

    n = int(1_000_000 * args.scale)
    g = int(np.ceil(np.sqrt(n)))
    xy, ro, go = synth.star_polygons(m=n, grid=g)
    a, b = upload(xy, ro, go), upload(xy + np.array([3.0, 2.0]), ro, go)
    out = torch.empty(n, dtype=torch.float64, device=dev)
    t = timed(st, lambda: E.check(lib.gpl_intersection_area(ctx._h, a._h, b._h, C.c_void_p(out.data_ptr()), None, E.GPL_DEVICE)), reps=3, warm=1)
    rec("intersection_area (%d star pairs, 64 x 64 edges)" % n, n, "row pairs", n * 64 * 64, t)
    del a, b

    sxy, sro, sgo = synth.star_polygons()
    stars = upload(sxy, sro, sgo)
    k = int(1000 * np.sqrt(args.scale))
    i, j = np.meshgrid(np.arange(k, dtype=np.float64), np.arange(k, dtype=np.float64), indexing="xy")
    x0, y0 = i.ravel() * (1000.0 / k), j.ravel() * (1000.0 / k)
    w = 1000.0 / k
    gxy = np.stack([np.stack([x0, x0 + w, x0 + w, x0, x0], 1), np.stack([y0, y0, y0 + w, y0 + w, y0], 1)], 2).reshape(-1, 2)
    cells = upload(gxy, np.arange(k * k + 1, dtype=np.int64) * 5, np.arange(k * k + 1, dtype=np.int64))
    n_pairs = [0]

    def join():
        h = C.c_void_p()
        E.check(lib.gpl_overlay_area_join(ctx._h, stars._h, cells._h, C.byref(h)))
        n_pairs[0] = int(lib.gpl_pairs_count(h))
        lib.gpl_pairs_free(h)

    t = timed(st, join, reps=3, warm=1)
    rec("overlay_area_join (10 000 stars x %d squares)" % (k * k), n_pairs[0], "pairs", n_pairs[0] * 64 * 4, t)


def boolean_rows(args, ctx, dev, st, res):
    """intersection, union and difference geometry (DESIGN.md §4.19) on the workload of overlay_rows: row-wise on 1 M pairs
    of config 2's stars against the same stars shifted by (3, 2), and the geometry overlay join of config 2's 10 000 stars
    against a 1000 x 1000 grid of unit squares; output MultiPolygon columns built on the device, host synchronisations of
    the count / scan / write passes included"""
    import numpy as np

    from geopolars_b200 import synth

    lib = ctx.lib

    def rec(name, units, unit_name, t, extra):
        r = {"op": name, "units": units, "unit": unit_name, "ms_min": t[0], "ms_avg": t[1], "units_per_s": units / (t[1] * 1e-3),
             "card": res["card"], "power_limit": res["power_limit"], **extra}
        res["rows"].append(r)
        print(json.dumps(r), flush=True)

    def upload(xy, ring_off, geom_off):
        t = [torch.from_numpy(np.ascontiguousarray(v)).to(dev) for v in (xy, ring_off, geom_off)]
        n = len(geom_off) - 1
        return ctx.wrap_device(GeometryType.POLYGON, n, len(xy), t[0].data_ptr(), geom_off_ptr=t[2].data_ptr(), ring_off_ptr=t[1].data_ptr(),
                               n_rings=len(ring_off) - 1, keepalive=tuple(t))

    n = int(1_000_000 * args.scale)
    g = int(np.ceil(np.sqrt(n)))
    xy, ro, go = synth.star_polygons(m=n, grid=g)
    a, b = upload(xy, ro, go), upload(xy + np.array([3.0, 2.0]), ro, go)
    for name, code in (("intersection", 0), ("union", 1), ("difference", 2)):
        size = [0]

        def run():
            h = C.c_void_p()
            E.check(lib.gpl_boolean_op(ctx._h, a._h, b._h, code, C.byref(h)))
            size[0] = int(E.DeviceArray(ctx, h).view().n_coords)

        t = timed(st, run, reps=3, warm=1)
        rec("boolean_op %s (%d star pairs, 64 x 64 edges)" % (name, n), n, "row pairs", t, {"out_coords": size[0]})
    del a, b

    sxy, sro, sgo = synth.star_polygons()
    stars = upload(sxy, sro, sgo)
    k = int(1000 * np.sqrt(args.scale))
    i, j = np.meshgrid(np.arange(k, dtype=np.float64), np.arange(k, dtype=np.float64), indexing="xy")
    x0, y0 = i.ravel() * (1000.0 / k), j.ravel() * (1000.0 / k)
    w = 1000.0 / k
    gxy = np.stack([np.stack([x0, x0 + w, x0 + w, x0, x0], 1), np.stack([y0, y0, y0 + w, y0 + w, y0], 1)], 2).reshape(-1, 2)
    cells = upload(gxy, np.arange(k * k + 1, dtype=np.int64) * 5, np.arange(k * k + 1, dtype=np.int64))
    n_pairs = [0]

    def join():
        hp, ha = C.c_void_p(), C.c_void_p()
        E.check(lib.gpl_overlay_join(ctx._h, stars._h, cells._h, C.byref(hp), C.byref(ha)))
        n_pairs[0] = int(lib.gpl_pairs_count(hp))
        lib.gpl_pairs_free(hp)
        E.DeviceArray(ctx, ha)

    t = timed(st, join, reps=3, warm=1)
    rec("overlay_join (10 000 stars x %d squares)" % (k * k), n_pairs[0], "pairs", t, {})


def phases(fn):
    """the GPU time of each kernel of one call of fn (torch.profiler), in ms, the 12 largest"""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = getattr(e, "cuda_time_total", 0.0)
        if t > 0:
            key = e.key.split("<")[0].split("(")[0].replace("void ", "").replace("gpl::", "")
            out[key] = round(out.get(key, 0.0) + t / 1e3, 3)
    return dict(sorted(out.items(), key=lambda kv: -kv[1])[:12])


def dissolve_rows(args, ctx, dev, st, res):
    """dissolve / union_all (DESIGN.md §4.21): 1 M two-row groups (config 2's stars and the same stars shifted by (3, 2)) beside
    the row-wise union of the same rows; the overlay round trip of the 10 000 stars (overlay_join with the 200 x 200 grid of
    5-unit squares, then dissolve of the pieces by star); union_all of the 10 000 stars plus the shifted stars (20 000 rows);
    union_all of naturalearth_lowres.  Each row also carries the per-kernel GPU time of one call (torch.profiler), so the
    phases (candidate join, nodes, classify, assembly) can be told apart."""
    import numpy as np

    from geopolars_b200 import datasets, synth

    lib = ctx.lib

    def rec(name, units, unit_name, t, extra):
        r = {"op": name, "units": units, "unit": unit_name, "ms_min": t[0], "ms_avg": t[1], "units_per_s": units / (t[1] * 1e-3),
             "card": res["card"], "power_limit": res["power_limit"], **extra}
        res["rows"].append(r)
        print(json.dumps(r), flush=True)

    def upload(xy, ring_off, geom_off):
        t = [torch.from_numpy(np.ascontiguousarray(v)).to(dev) for v in (xy, ring_off, geom_off)]
        n = len(geom_off) - 1
        return ctx.wrap_device(GeometryType.POLYGON, n, len(xy), t[0].data_ptr(), geom_off_ptr=t[2].data_ptr(), ring_off_ptr=t[1].data_ptr(),
                               n_rings=len(ring_off) - 1, keepalive=tuple(t))

    def pair_column(xy, ro):
        n = len(ro) - 1
        return upload(np.concatenate([xy, xy + np.array([3.0, 2.0])]), np.concatenate([ro, ro[1:] + ro[-1]]), np.arange(2 * n + 1, dtype=np.int64))

    def dissolve_call(col, codes, ng, size):
        def run():
            h = C.c_void_p()
            E.check(lib.gpl_dissolve(ctx._h, col._h, codes.ctypes.data, E.GPL_HOST, ng, C.byref(h)))
            size[0] = int(E.DeviceArray(ctx, h).view().n_coords)
        return run

    n = int(1_000_000 * args.scale)
    g = int(np.ceil(np.sqrt(n)))
    xy, ro, go = synth.star_polygons(m=n, grid=g)
    a, b = upload(xy, ro, go), upload(xy + np.array([3.0, 2.0]), ro, go)
    size = [0]

    def union():
        h = C.c_void_p()
        E.check(lib.gpl_boolean_op(ctx._h, a._h, b._h, 1, C.byref(h)))
        size[0] = int(E.DeviceArray(ctx, h).view().n_coords)

    t = timed(st, union, reps=3, warm=1)
    rec("boolean_op union (%d star pairs, 64 x 64 edges)" % n, n, "row pairs", t, {"out_coords": size[0]})
    del a, b
    both = pair_column(xy, ro)
    codes = np.concatenate([np.arange(n), np.arange(n)]).astype(np.int64)
    run = dissolve_call(both, codes, n, size)
    t = timed(st, run, reps=3, warm=1)
    rec("dissolve (%d two-row star groups)" % n, n, "groups", t, {"out_coords": size[0], "phases_ms": phases(run)})
    del both

    sxy, sro, sgo = synth.star_polygons()
    stars = upload(sxy, sro, sgo)
    k = 200
    i, j = np.meshgrid(np.arange(k, dtype=np.float64), np.arange(k, dtype=np.float64), indexing="xy")
    x0, y0 = i.ravel() * 5.0, j.ravel() * 5.0
    gxy = np.stack([np.stack([x0, x0 + 5.0, x0 + 5.0, x0, x0], 1), np.stack([y0, y0, y0 + 5.0, y0 + 5.0, y0], 1)], 2).reshape(-1, 2)
    cells = upload(gxy, np.arange(k * k + 1, dtype=np.int64) * 5, np.arange(k * k + 1, dtype=np.int64))
    li, _, pieces = E.overlay_join(stars, cells)
    lcodes = li.astype(np.int64)
    run = dissolve_call(pieces, lcodes, len(sgo) - 1, size)
    t = timed(st, run, reps=3, warm=1)
    rec("dissolve (overlay round trip: %d pieces of 10 000 stars)" % len(li), len(li), "rows", t, {"out_coords": size[0], "phases_ms": phases(run)})

    for m, grid in ((300, 20), (1000, 40)):  # one group is assembled by one thread: its cost grows faster than its size
        mxy, mro, _ = synth.star_polygons(m=m, grid=grid)
        both = pair_column(mxy, mro)
        zeros = np.zeros(len(both), dtype=np.int64)
        run = dissolve_call(both, zeros, 1, size)
        t = timed(st, run, reps=1, warm=0)
        rec("union_all (%d stars + the same shifted by (3, 2))" % m, len(both), "rows", t, {"out_coords": size[0], "phases_ms": phases(run)})

    ne = datasets.read_dataset("naturalearth_lowres").geometry.device
    zeros = np.zeros(len(ne), dtype=np.int64)
    run = dissolve_call(ne, zeros, 1, size)
    t = timed(st, run, reps=3, warm=1)
    rec("union_all (naturalearth_lowres, %d rows)" % len(ne), len(ne), "rows", t, {"out_coords": size[0], "phases_ms": phases(run)})


def overlay_modes_rows(args, ctx, dev, st, res):
    """symmetric difference and the overlay modes (DESIGN.md §4.23): the row-wise symmetric difference of 1 M pairs of config
    2's stars against the same stars shifted by (3, 2), beside the row-wise union of the same pairs; overlay in all five modes
    of config 2's 10 000 stars against the same stars shifted by (3, 2); identity of naturalearth_lowres against the 5-degree
    grid; difference of one large polygon (a 256-gon of radius 220 over the middle of 2 000 stars spread over 450 x 450) against
    those stars, one remainder with about 1 500 cutters, which one thread assembles.  Each row carries the per-kernel GPU time of one call (torch.profiler)."""
    import numpy as np

    from geopolars_b200 import datasets, synth

    lib = ctx.lib

    def rec(name, units, unit_name, t, extra):
        r = {"op": name, "units": units, "unit": unit_name, "ms_min": t[0], "ms_avg": t[1], "units_per_s": units / (t[1] * 1e-3),
             "card": res["card"], "power_limit": res["power_limit"], **extra}
        res["rows"].append(r)
        print(json.dumps(r), flush=True)

    def upload(xy, ring_off, geom_off):
        t = [torch.from_numpy(np.ascontiguousarray(v)).to(dev) for v in (xy, ring_off, geom_off)]
        n = len(geom_off) - 1
        return ctx.wrap_device(GeometryType.POLYGON, n, len(xy), t[0].data_ptr(), geom_off_ptr=t[2].data_ptr(), ring_off_ptr=t[1].data_ptr(),
                               n_rings=len(ring_off) - 1, keepalive=tuple(t))

    def boolean_call(a, b, code, size):
        def run():
            h = C.c_void_p()
            E.check(lib.gpl_boolean_op(ctx._h, a._h, b._h, code, C.byref(h)))
            size[0] = int(E.DeviceArray(ctx, h).view().n_coords)
        return run

    def overlay_call(lhs, rhs, how, size):
        def run():
            hp, ha = C.c_void_p(), C.c_void_p()
            E.check(lib.gpl_overlay(ctx._h, lhs._h, rhs._h, E.OVERLAY_HOWS[how], C.byref(hp), C.byref(ha)))
            size[0] = int(lib.gpl_pairs_count(hp))
            lib.gpl_pairs_free(hp)
            E.DeviceArray(ctx, ha)
        return run

    size = [0]
    n = int(1_000_000 * args.scale)
    g = int(np.ceil(np.sqrt(n)))
    xy, ro, go = synth.star_polygons(m=n, grid=g)
    a, b = upload(xy, ro, go), upload(xy + np.array([3.0, 2.0]), ro, go)
    for name, code in (("symmetric_difference", 3), ("union", 1)):
        run = boolean_call(a, b, code, size)
        t = timed(st, run, reps=3, warm=1)
        rec("boolean_op %s (%d star pairs, 64 x 64 edges)" % (name, n), n, "row pairs", t, {"out_coords": size[0], "phases_ms": phases(run)})
    del a, b

    sxy, sro, sgo = synth.star_polygons()
    stars, shifted = upload(sxy, sro, sgo), upload(sxy + np.array([3.0, 2.0]), sro, sgo)
    for how in ("intersection", "union", "identity", "symmetric_difference", "difference"):
        run = overlay_call(stars, shifted, how, size)
        t = timed(st, run, reps=3, warm=1)
        rec("overlay %s (10 000 stars x the same shifted by (3, 2))" % how, size[0], "rows", t, {"phases_ms": phases(run)})

    k = 72 * 36
    i, j = np.meshgrid(np.arange(72, dtype=np.float64), np.arange(36, dtype=np.float64), indexing="xy")
    x0, y0 = -180.0 + i.ravel() * 5.0, -90.0 + j.ravel() * 5.0
    gxy = np.stack([np.stack([x0, x0 + 5.0, x0 + 5.0, x0, x0], 1), np.stack([y0, y0, y0 + 5.0, y0 + 5.0, y0], 1)], 2).reshape(-1, 2)
    cells = upload(gxy, np.arange(k + 1, dtype=np.int64) * 5, np.arange(k + 1, dtype=np.int64))
    ne = datasets.read_dataset("naturalearth_lowres").geometry.device
    run = overlay_call(ne, cells, "identity", size)
    t = timed(st, run, reps=3, warm=1)
    rec("overlay identity (naturalearth_lowres x the 5-degree grid)", size[0], "rows", t, {"phases_ms": phases(run)})

    mxy, mro, mgo = synth.star_polygons(m=2000, grid=45)
    few = upload(mxy, mro, mgo)
    c = mxy.min(0) + (mxy.max(0) - mxy.min(0)) / 2
    ang = np.arange(256) * (2 * np.pi / 256)
    big_xy = np.concatenate([np.stack([c[0] + 220 * np.cos(ang), c[1] + 220 * np.sin(ang)], 1), [[c[0] + 220, c[1]]]])
    big = upload(big_xy, np.array([0, 257], dtype=np.int64), np.array([0, 1], dtype=np.int64))
    pl, _ = E.spatial_join(big, few, "intersects")
    run = overlay_call(big, few, "difference", size)
    t = timed(st, run, reps=1, warm=0)
    rec("overlay difference (one 256-gon x 2 000 stars, %d cutters)" % len(pl), 1, "remainders", t, {"phases_ms": phases(run)})


def relate_rows(args, ctx, dev, st, res):
    """DE-9IM (DESIGN.md §4.20) on the workload of boolean_rows: relate and the touches / within predicates row-wise on 1 M
    pairs of config 2's stars against the same stars shifted by (3, 2); the predicate join of config 2's 10 000 stars against
    a 1000 x 1000 grid of unit squares for intersects, touches and within (candidates, sort and the per-pair kernel, host
    synchronisations included); points within polygons, 10 M uniform points against the 10 000 stars, through the
    points-in-polygons index and through the DE-9IM route"""
    import numpy as np

    from geopolars_b200 import synth

    lib = ctx.lib

    def rec(name, units, unit_name, t, extra):
        r = {"op": name, "units": units, "unit": unit_name, "ms_min": t[0], "ms_avg": t[1], "units_per_s": units / (t[1] * 1e-3),
             "card": res["card"], "power_limit": res["power_limit"], **extra}
        res["rows"].append(r)
        print(json.dumps(r), flush=True)

    def upload(xy, ring_off, geom_off):
        t = [torch.from_numpy(np.ascontiguousarray(v)).to(dev) for v in (xy, ring_off, geom_off)]
        n = len(geom_off) - 1
        return ctx.wrap_device(GeometryType.POLYGON, n, len(xy), t[0].data_ptr(), geom_off_ptr=t[2].data_ptr(), ring_off_ptr=t[1].data_ptr(),
                               n_rings=len(ring_off) - 1, keepalive=tuple(t))

    n = int(1_000_000 * args.scale)
    g = int(np.ceil(np.sqrt(n)))
    xy, ro, go = synth.star_polygons(m=n, grid=g)
    a, b = upload(xy, ro, go), upload(xy + np.array([3.0, 2.0]), ro, go)
    mat = torch.empty(n * 9, dtype=torch.int8, device=dev)
    bits = torch.empty((n + 7) // 8, dtype=torch.uint8, device=dev)
    t = timed(st, lambda: E.check(lib.gpl_relate(ctx._h, a._h, b._h, C.c_void_p(mat.data_ptr()), None, E.GPL_DEVICE)), reps=3, warm=1)
    rec("relate (%d star pairs, 64 x 64 edges)" % n, n, "row pairs", t, {})
    for name in ("touches", "within"):
        code = E.RELATE_PREDICATES[name]
        t = timed(st, lambda: E.check(lib.gpl_relate_predicate(ctx._h, a._h, b._h, code, None, C.c_void_p(bits.data_ptr()), E.GPL_DEVICE)),
                  reps=3, warm=1)
        rec("relate_predicate %s (%d star pairs)" % (name, n), n, "row pairs", t, {})
    del a, b

    sxy, sro, sgo = synth.star_polygons()
    stars = upload(sxy, sro, sgo)
    k = int(1000 * np.sqrt(args.scale))
    i, j = np.meshgrid(np.arange(k, dtype=np.float64), np.arange(k, dtype=np.float64), indexing="xy")
    x0, y0 = i.ravel() * (1000.0 / k), j.ravel() * (1000.0 / k)
    w = 1000.0 / k
    gxy = np.stack([np.stack([x0, x0 + w, x0 + w, x0, x0], 1), np.stack([y0, y0, y0 + w, y0 + w, y0], 1)], 2).reshape(-1, 2)
    cells = upload(gxy, np.arange(k * k + 1, dtype=np.int64) * 5, np.arange(k * k + 1, dtype=np.int64))

    def join(lhs, rhs, code, out):
        h = C.c_void_p()
        E.check(lib.gpl_predicate_join(ctx._h, lhs._h, rhs._h, code, None, C.byref(h)))
        out[0] = int(lib.gpl_pairs_count(h))
        lib.gpl_pairs_free(h)

    for name, lhs, rhs in (("intersects", stars, cells), ("touches", stars, cells), ("within", cells, stars)):
        cnt = [0]
        t = timed(st, lambda: join(lhs, rhs, E.RELATE_PREDICATES[name], cnt), reps=3, warm=1)
        rec("predicate_join %s (%d x %d)" % (name, len(lhs), len(rhs)), cnt[0], "pairs", t, {})

    m = int(10_000_000 * args.scale)
    pts_t = torch.empty((m, 2), dtype=torch.float64, device=dev)
    E.check(lib.gpl_gen_uniform_points(ctx._h, 9, 0, m, 1000.0, pts_t.data_ptr()))
    pts = ctx.wrap_device(GeometryType.POINT, m, m, pts_t.data_ptr(), keepalive=(pts_t,))
    cnt = [0]

    def pip():
        idx = E.PipIndex(stars)
        h = C.c_void_p()
        E.check(lib.gpl_contains_join_pairs_array(ctx._h, idx._h, pts._h, C.byref(h)))
        cnt[0] = int(lib.gpl_pairs_count(h))
        lib.gpl_pairs_free(h)
        idx.free()

    t = timed(st, pip, reps=3, warm=1)
    rec("points within polygons, index route (%d points x %d stars, index build included)" % (m, len(stars)), cnt[0], "pairs", t, {})
    t = timed(st, lambda: join(pts, stars, E.RELATE_PREDICATES["within"], cnt), reps=3, warm=1)
    rec("points within polygons, relate route (%d points x %d stars)" % (m, len(stars)), cnt[0], "pairs", t, {})


def clip_rows(args, ctx, dev, st, res):
    """line clipping (DESIGN.md §4.22): clip, clip(invert) and clip_length of 1 M config-3 walks (16 coordinates), each
    against config 2's star whose 10 m cell holds the walk's start, with relate on the same row pairs for context; the
    length-weighted overlay join of the 1 M walks against the 10 000 stars and of 100 000 walks against a 1000 x 1000 grid
    of unit squares (candidates, sort and the per-pair kernels, host synchronisations included)"""
    import numpy as np

    from geopolars_b200 import synth

    lib = ctx.lib

    def rec(name, units, unit_name, t, extra):
        r = {"op": name, "units": units, "unit": unit_name, "ms_min": t[0], "ms_avg": t[1], "units_per_s": units / (t[1] * 1e-3),
             "card": res["card"], "power_limit": res["power_limit"], **extra}
        res["rows"].append(r)
        print(json.dumps(r), flush=True)

    def polygons(xy_t, ring_off, geom_off):
        t = [torch.from_numpy(np.ascontiguousarray(v)).to(dev) for v in (ring_off, geom_off)]
        n = len(geom_off) - 1
        return ctx.wrap_device(GeometryType.POLYGON, n, xy_t.shape[0], xy_t.data_ptr(), geom_off_ptr=t[1].data_ptr(), ring_off_ptr=t[0].data_ptr(),
                               n_rings=len(ring_off) - 1, keepalive=(xy_t, *t))

    def walks(n, stream):
        xy = torch.empty((n * 16, 2), dtype=torch.float64, device=dev)
        off = torch.empty(n + 1, dtype=torch.int64, device=dev)
        E.check(lib.gpl_gen_walk_linestrings(ctx._h, stream, -1, 0, n, 16, xy.data_ptr(), off.data_ptr()))
        return xy, ctx.wrap_device(GeometryType.LINESTRING, n, n * 16, xy.data_ptr(), geom_off_ptr=off.data_ptr(), keepalive=(xy, off))

    n = int(1_000_000 * args.scale)
    wxy, lines = walks(n, 3)
    sxy, sro, sgo = synth.star_polygons()
    stars_t = torch.from_numpy(sxy).to(dev)
    start = wxy.view(n, 16, 2)[:, 0, :]
    cell = (torch.clamp(torch.floor(start[:, 1] / 10.0), 0, 99) * 100 + torch.clamp(torch.floor(start[:, 0] / 10.0), 0, 99)).long()
    mine = stars_t.view(-1, 65, 2)[cell].reshape(-1, 2).contiguous()
    polys = polygons(mine, np.arange(n + 1, dtype=np.int64) * 65, np.arange(n + 1, dtype=np.int64))
    out = torch.empty(n, dtype=torch.float64, device=dev)
    mat = torch.empty(n * 9, dtype=torch.int8, device=dev)
    for inv in (0, 1):
        coords = [0]

        def run():
            h = C.c_void_p()
            E.check(lib.gpl_clip(ctx._h, lines._h, polys._h, inv, C.byref(h)))
            d = E.DeviceArray(ctx, h)
            coords[0] = int(d.view().n_coords)
            d.free()

        t = timed(st, run, reps=3, warm=1)
        rec("clip%s (%d walks x their cell's star, 15 x 64 edges)" % (" invert" if inv else "", n), n, "row pairs", t, {"out_coords": coords[0]})
    t = timed(st, lambda: E.check(lib.gpl_clip_length(ctx._h, lines._h, polys._h, C.c_void_p(out.data_ptr()), None, E.GPL_DEVICE)), reps=3, warm=1)
    rec("clip_length (%d walks x their cell's star)" % n, n, "row pairs", t, {"total_length": float(out.sum().item())})
    t = timed(st, lambda: E.check(lib.gpl_relate(ctx._h, lines._h, polys._h, C.c_void_p(mat.data_ptr()), None, E.GPL_DEVICE)), reps=3, warm=1)
    rec("relate (the same %d row pairs)" % n, n, "row pairs", t, {})
    del polys, mine

    def join(lhs, rhs, out):
        h = C.c_void_p()
        E.check(lib.gpl_overlay_length_join(ctx._h, lhs._h, rhs._h, C.byref(h)))
        out[0] = int(lib.gpl_pairs_count(h))
        lib.gpl_pairs_free(h)

    stars = polygons(stars_t, sro, sgo)
    cnt = [0]
    t = timed(st, lambda: join(lines, stars, cnt), reps=3, warm=1)
    rec("overlay_length_join (%d walks x 10 000 stars)" % n, cnt[0], "pairs", t, {})
    m = int(100_000 * args.scale)
    _, few = walks(m, 4)
    k = int(1000 * np.sqrt(args.scale))
    i, j = np.meshgrid(np.arange(k, dtype=np.float64), np.arange(k, dtype=np.float64), indexing="xy")
    x0, y0 = i.ravel() * (1000.0 / k), j.ravel() * (1000.0 / k)
    w = 1000.0 / k
    gxy = np.stack([np.stack([x0, x0 + w, x0 + w, x0, x0], 1), np.stack([y0, y0, y0 + w, y0 + w, y0], 1)], 2).reshape(-1, 2)
    cells = polygons(torch.from_numpy(gxy).to(dev), np.arange(k * k + 1, dtype=np.int64) * 5, np.arange(k * k + 1, dtype=np.int64))
    t = timed(st, lambda: join(few, cells, cnt), reps=3, warm=1)
    rec("overlay_length_join (%d walks x %d unit squares)" % (m, k * k), cnt[0], "pairs", t, {})


def geodesic_rows(args, ctx, dev, st, res):
    """geodesic area and perimeter on WGS84 (DESIGN.md §4.17), kernel resident, one call filling both outputs: 1 M config-2
    stars (65 coordinates, 65 edges each) mapped to (lon, lat) with radii near 0.01 degrees over |lat| <= 80, 10 M closed
    5-coordinate parcels (about 20 m), and naturalearth_lowres repeated to about 1 M rows.  ms, rows/s and edges/s (an edge is
    one inverse solve with the area term: FP64 and transcendental bound).  The CPU arm is the C oracle with every core
    (threads=0) on the first 10 % of the rows of each input: og_geodesic_length(method="geodesic") runs the same Karney
    inverse solve for every edge of the exterior rings, without the area term, so its edges/s bound what a CPU area pass
    could reach from above."""
    import time

    import numpy as np

    from geopolars_b200 import datasets, synth

    from oracle import oracle as og

    lib = ctx.lib
    rng = np.random.default_rng(2024)

    def rec(name, rows, edges, t, cpu_edges_per_s):
        r = {"op": name, "units": rows, "unit": "rows", "ms_min": t[0], "ms_avg": t[1], "units_per_s": rows / (t[1] * 1e-3),
             "edges": edges, "edges_per_s": edges / (t[1] * 1e-3), "cpu_oracle_threads": og.max_threads(), "cpu_oracle_edges_per_s": cpu_edges_per_s,
             "card": res["card"], "power_limit": res["power_limit"]}
        res["rows"].append(r)
        print(json.dumps(r), flush=True)

    def upload(type_, xy, ring_off, geom_off, part_off=None):
        vs = [xy, ring_off, geom_off] + ([part_off] if part_off is not None else [])
        t = [torch.from_numpy(np.ascontiguousarray(v)).to(dev) for v in vs]
        return ctx.wrap_device(type_, len(geom_off) - 1, len(xy), t[0].data_ptr(), geom_off_ptr=t[2].data_ptr(), ring_off_ptr=t[1].data_ptr(),
                               part_off_ptr=t[3].data_ptr() if part_off is not None else None, n_rings=len(ring_off) - 1,
                               n_parts=len(part_off) - 1 if part_off is not None else 0, keepalive=tuple(t))

    def cpu_rate(type_, xy, ring_off, geom_off, part_off):
        """C oracle (threads=0) Karney solves per second over the exterior-ring edges of the first 10 % of the rows"""
        k = max(1, (len(geom_off) - 1) // 10)
        go = geom_off[: k + 1]
        if type_ == GeometryType.MULTIPOLYGON:
            po = part_off[: go[-1] + 1]
            ro = ring_off[: po[-1] + 1]
            exterior = po[:-1][po[1:] > po[:-1]]
            a = og.OGArray(og.MULTIPOLYGON, xy[: ro[-1]], geom_off=go, part_off=po, ring_off=ro)
        else:
            ro = ring_off[: go[-1] + 1]
            exterior = go[:-1][go[1:] > go[:-1]]
            a = og.OGArray(og.POLYGON, xy[: ro[-1]], geom_off=go, ring_off=ro)
        edges = int(np.maximum(ro[exterior + 1] - ro[exterior] - 1, 0).sum())
        og.geodesic_length(a, "geodesic", threads=0)  # warm-up: loads the library and starts the threads
        t0 = time.perf_counter()
        og.geodesic_length(a, "geodesic", threads=0)
        return edges / (time.perf_counter() - t0)

    def measure(name, type_, xy, ring_off, geom_off, part_off=None):
        a = upload(type_, xy, ring_off, geom_off, part_off)
        n = len(geom_off) - 1
        area = torch.empty(n, dtype=torch.float64, device=dev)
        per = torch.empty(n, dtype=torch.float64, device=dev)
        t = timed(st, lambda: E.check(lib.gpl_geodesic_area(ctx._h, a._h, 1, C.c_void_p(area.data_ptr()), C.c_void_p(per.data_ptr()), None,
                                                            E.GPL_DEVICE)), reps=3, warm=1)
        rec(name, n, len(xy), t, cpu_rate(type_, xy, ring_off, geom_off, part_off))
        del a, area, per
        torch.cuda.empty_cache()

    n = int(1_000_000 * args.scale)
    g = int(np.ceil(np.sqrt(n)))
    xy, ro, go = synth.star_polygons(m=n, grid=g)
    c = (xy[ro[:-1]] + xy[ro[:-1] + 32]) / 2  # centre of each star (vertex 0 and 32 are opposite)
    ll = np.stack([rng.uniform(-180, 180, n), rng.uniform(-80, 80, n)], 1)
    xy = (np.repeat(ll, 65, 0) + (xy - np.repeat(c, 65, 0)) * (0.01 / 4.0))
    measure("geodesic_area (%d stars, 65 coordinates, r ~ 0.01 deg)" % n, GeometryType.POLYGON, xy, ro, go)
    del xy

    n = int(10_000_000 * args.scale)
    ll = np.stack([rng.uniform(-180, 180, n), rng.uniform(-80, 80, n)], 1)
    d = 0.0002 * rng.uniform(0.5, 1.5, (n, 2))
    q = np.empty((n, 5, 2))
    q[:, 0] = ll
    q[:, 1] = ll + [1, 0] * d
    q[:, 2] = ll + d
    q[:, 3] = ll + [0, 1] * d
    q[:, 4] = ll
    measure("geodesic_area (%d parcels, 5 coordinates, ~20 m)" % n, GeometryType.POLYGON, q.reshape(-1, 2), np.arange(n + 1, dtype=np.int64) * 5,
            np.arange(n + 1, dtype=np.int64))
    del q

    h = datasets.read_dataset("naturalearth_lowres").geometry.device.to_host()
    reps = max(1, int(round(1_000_000 * args.scale / len(h.geom_off[:-1]))))
    h_part = h.part_off if h.type == GeometryType.MULTIPOLYGON else np.arange(len(h.geom_off), dtype=np.int64)
    h_geom = h.geom_off if h.type == GeometryType.MULTIPOLYGON else np.arange(len(h.geom_off), dtype=np.int64)
    nc, nr, npart = len(h.xy), len(h.ring_off) - 1, len(h_part) - 1
    xy = np.tile(h.xy, (reps, 1))
    ro = np.concatenate([h.ring_off[:-1] + k * nc for k in range(reps)] + [[reps * nc]]).astype(np.int64)
    po = np.concatenate([(h_part if h.type == GeometryType.MULTIPOLYGON else h.geom_off)[:-1] + k * nr for k in range(reps)] + [[reps * nr]]).astype(np.int64)
    go = np.concatenate([h_geom[:-1] + k * npart for k in range(reps)] + [[reps * npart]]).astype(np.int64)
    measure("geodesic_area (naturalearth_lowres x %d, %d rows)" % (reps, len(go) - 1), GeometryType.MULTIPOLYGON, xy, ro, go, po)


def valid_rows(args, ctx, dev, st, res):
    """OGC validity (DESIGN.md §4.18), kernel resident, reason codes to device memory: 1 M config-2 stars (65 coordinates),
    10 M closed 5-coordinate parcels, naturalearth_lowres repeated to about 1 M rows, one 10^6-vertex regular polygon and one
    square with 10 000 square holes.  ms, rows/s and edges/s (an edge is one ring edge of the input; the edge-pair pass tests
    each against the edges of the candidate chunks its grid cell lists: FP64 orientation bound)."""
    import numpy as np

    from geopolars_b200 import datasets, synth

    lib = ctx.lib

    def measure(name, type_, xy, ring_off, geom_off, part_off=None):
        vs = [xy, ring_off, geom_off] + ([part_off] if part_off is not None else [])
        t = [torch.from_numpy(np.ascontiguousarray(v)).to(dev) for v in vs]
        a = ctx.wrap_device(type_, len(geom_off) - 1, len(xy), t[0].data_ptr(), geom_off_ptr=t[2].data_ptr(), ring_off_ptr=t[1].data_ptr(),
                            part_off_ptr=t[3].data_ptr() if part_off is not None else None, n_rings=len(ring_off) - 1,
                            n_parts=len(part_off) - 1 if part_off is not None else 0, keepalive=tuple(t))
        n = len(geom_off) - 1
        out = torch.empty(n, dtype=torch.int8, device=dev)
        tm = timed(st, lambda: E.check(lib.gpl_is_valid(ctx._h, a._h, C.c_void_p(out.data_ptr()), None, E.GPL_DEVICE)), reps=5, warm=2)
        edges = len(xy) - (len(ring_off) - 1)  # closed rings
        r = {"op": name, "units": n, "unit": "rows", "ms_min": tm[0], "ms_avg": tm[1], "units_per_s": n / (tm[1] * 1e-3), "edges": edges,
             "edges_per_s": edges / (tm[1] * 1e-3), "invalid_rows": int((out != 0).sum().item()), "card": res["card"], "power_limit": res["power_limit"]}
        res["rows"].append(r)
        print(json.dumps(r), flush=True)

    m = int(1_000_000 * args.scale)
    xy, ro, go = synth.star_polygons(m, int(np.ceil(np.sqrt(m))))
    measure("is_valid (%d config-2 stars)" % m, GeometryType.POLYGON, xy, ro, go)
    del xy
    n = int(10_000_000 * args.scale)
    k = int(np.ceil(np.sqrt(n)))
    ll = np.stack([np.arange(n) % k, np.arange(n) // k], 1).astype(np.float64) * 2.0
    q = np.empty((n, 5, 2))
    q[:, 0], q[:, 1], q[:, 2], q[:, 3], q[:, 4] = ll, ll + [1, 0], ll + 1, ll + [0, 1], ll
    measure("is_valid (%d parcels, 5 coordinates)" % n, GeometryType.POLYGON, q.reshape(-1, 2), np.arange(n + 1, dtype=np.int64) * 5,
            np.arange(n + 1, dtype=np.int64))
    del q, ll
    h = datasets.read_dataset("naturalearth_lowres").geometry.device.to_host()
    reps = max(1, int(round(1_000_000 * args.scale / len(h.geom_off[:-1]))))
    h_part = h.part_off if h.type == GeometryType.MULTIPOLYGON else np.arange(len(h.geom_off), dtype=np.int64)
    h_geom = h.geom_off if h.type == GeometryType.MULTIPOLYGON else np.arange(len(h.geom_off), dtype=np.int64)
    nc, nr, npart = len(h.xy), len(h.ring_off) - 1, len(h_part) - 1
    ro = np.concatenate([h.ring_off[:-1] + i * nc for i in range(reps)] + [[reps * nc]]).astype(np.int64)
    po = np.concatenate([h_part[:-1] + i * nr for i in range(reps)] + [[reps * nr]]).astype(np.int64)
    go = np.concatenate([h_geom[:-1] + i * npart for i in range(reps)] + [[reps * npart]]).astype(np.int64)
    measure("is_valid (naturalearth_lowres x %d, %d rows)" % (reps, len(go) - 1), GeometryType.MULTIPOLYGON, np.tile(h.xy, (reps, 1)), ro, go, po)
    nv = 1_000_000
    t = 2 * np.pi * np.arange(nv + 1) / nv
    ring = np.stack([np.cos(t), np.sin(t)], 1) * 1000.0
    ring[-1] = ring[0]
    measure("is_valid (one ring of %d vertices)" % nv, GeometryType.POLYGON, ring, np.array([0, nv + 1]), np.array([0, 1]))
    g = 100
    holes = [np.array([[0, 0], [301, 0], [301, 301], [0, 301], [0, 0]], float)]
    holes += [np.array([[x, y], [x, y + 1], [x + 1, y + 1], [x + 1, y], [x, y]], float) for x in range(1, 3 * g, 3) for y in range(1, 3 * g, 3)]
    measure("is_valid (one polygon with %d holes)" % (g * g), GeometryType.POLYGON, np.concatenate(holes), np.arange(len(holes) + 1) * 5,
            np.array([0, len(holes)]))


def geo_rows(args, ctx, dev, st, res):
    """great-circle joins (DESIGN.md §4.15), kernel resident: build ms, count-pass ms, pair-list ms (with distances), dense
    nearest ms; left rows/s, pairs/s, exact haversine evaluations per left row and per second.  An evaluation is 2 sin, 1
    sqrt, 1 asin and about 15 FP64 operations on one 32-byte record: the kernels are FP64 / transcendental bound, not HBM
    bound (evaluations/s x 32 B is far below the HBM peak).  Plus a cKDTree CPU arm on unit vectors for workload 1."""
    import time

    import numpy as np

    lib = ctx.lib
    D = 1e4

    def upload(P):
        t = torch.from_numpy(np.ascontiguousarray(P)).to(dev)
        return ctx.wrap_device(GeometryType.POINT, len(P), len(P), t.data_ptr(), keepalive=(t,))

    def run(name, L, Rr):
        lhs, rhs, n = upload(L), upload(Rr), len(L)
        tb = timed(st, lambda: E.GeoIndex(rhs).free(), reps=3, warm=1)
        idx = E.GeoIndex(rhs)
        cnt = torch.empty(n, dtype=torch.int32, device=dev)
        tc = timed(st, lambda: E.check(lib.gpl_geo_dwithin_count(ctx._h, idx._h, lhs._h, D, C.c_void_p(cnt.data_ptr()), E.GPL_DEVICE)), reps=3, warm=1)
        evals = idx.stats()["evaluations"]
        n_pairs = [0]

        def pairs():
            h = C.c_void_p()
            E.check(lib.gpl_geo_dwithin_join_pairs(ctx._h, idx._h, lhs._h, D, 1, C.byref(h)))
            n_pairs[0] = int(lib.gpl_pairs_count(h))
            lib.gpl_pairs_free(h)

        tp = timed(st, pairs, reps=3, warm=1)
        nid = torch.empty(n, dtype=torch.int32, device=dev)
        dist = torch.empty(n, dtype=torch.float64, device=dev)
        tn = timed(st, lambda: E.check(lib.gpl_geo_nearest_join(ctx._h, idx._h, lhs._h, float("inf"), C.c_void_p(nid.data_ptr()),
                                                                C.c_void_p(dist.data_ptr()), None, E.GPL_DEVICE)), reps=3, warm=1)
        s = idx.stats()
        r = {"op": f"great-circle joins: {name}, D = {D} m", "left_rows": n, "rhs_rows": len(Rr), "build_ms_min": tb[0],
             "count_ms_min": tc[0], "count_ms_avg": tc[1], "pairs_ms_min": tp[0], "pairs_ms_avg": tp[1], "nearest_ms_min": tn[0],
             "nearest_ms_avg": tn[1], "count_left_rows_per_s": n / (tc[1] * 1e-3), "pairs_left_rows_per_s": n / (tp[1] * 1e-3),
             "pairs_per_s": n_pairs[0] / (tp[1] * 1e-3), "nearest_left_rows_per_s": n / (tn[1] * 1e-3), "pairs": n_pairs[0],
             "count_evals_per_left_row": evals / n, "count_evals_per_s": evals / (tc[1] * 1e-3),
             "count_item_GBps": evals * 32 / (tc[1] * 1e-3) / 1e9, "nearest_evals_per_left_row": s["evaluations"] / n,
             "nearest_evals_per_s": s["evaluations"] / (tn[1] * 1e-3), "grid_cells_per_axis": s["grid_cells_per_axis"],
             "card": res["card"], "power_limit": res["power_limit"]}
        idx.free()
        res["rows"].append(r)
        print(json.dumps(r), flush=True)

    def sphere(rng, n):
        return np.column_stack([rng.uniform(-180, 180, n), np.degrees(np.arcsin(rng.uniform(-1, 1, n)))])

    NP, NR = int(10_000_000 * max(args.scale, 0.01)), int(1_000_000 * max(args.scale, 0.01))
    rng = np.random.default_rng(415)
    L, Rr = sphere(rng, NP), sphere(rng, NR)
    run(f"{NP} x {NR} points uniform on the sphere", L, Rr)
    # real data is skewed: both sides scattered about 100 km (1 degree sigma in latitude) around the naturalearth_cities rows
    from geopolars_b200 import datasets

    c = datasets.read_dataset("naturalearth_cities").geometry.device.to_host().xy

    def around(n):
        k = c[rng.integers(0, len(c), n)]
        lat = np.clip(k[:, 1] + rng.normal(0, 0.9, n), -89.9, 89.9)
        return np.column_stack([k[:, 0] + rng.normal(0, 0.9, n) / np.cos(np.radians(lat)), lat])

    run(f"{NP} x {NR} points clustered around {len(c)} cities", around(NP), around(NR))
    # CPU arm of workload 1: cKDTree on 3-D unit vectors, chord radius 2 sin(D / 2R), a prefix of the left points
    from scipy.spatial import cKDTree

    def unit(P):
        lo, la = np.radians(P[:, 0]), np.radians(P[:, 1])
        return np.column_stack([np.cos(la) * np.cos(lo), np.cos(la) * np.sin(lo), np.sin(la)])

    k = min(NP, 2_000_000)
    t0 = time.perf_counter()
    tree = cKDTree(unit(Rr))
    t1 = time.perf_counter()
    nb = tree.query_ball_point(unit(L[:k]), 2.0 * np.sin(D / 6371008.8 / 2.0), workers=-1, return_length=True)
    t2 = time.perf_counter()
    r = {"op": f"great-circle dwithin CPU arm: scipy cKDTree.query_ball_point(workers=-1, return_length=True) on unit vectors, {k}-point "
               "prefix of workload 1 (candidate counts by chord: no haversine evaluation)",
         "left_rows": k, "nproc": os.cpu_count(), "build_s": t1 - t0, "query_s": t2 - t1, "left_rows_per_s": k / (t2 - t1), "pairs": int(nb.sum())}
    res["rows"].append(r)
    print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
