#!/usr/bin/env python
"""Kernel-resident timings of the other §8 rows at BASELINE config sizes (3 and 5), with the HBM roofline
fraction for the coordinate bytes read, and of the nearest join (100 M points against config 2's polygons, 1 M
reference points and 1 M walk linestrings).  Not the flagship bench (that is bench.py, config 2); config 5 runs at
4 M polygons so that its input and output columns fit one 80 GB H100.

  python tools/bench_ops.py [--scale 1.0] [--only all|ops|nearest] [--out ops_roofline.json]
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
    ap.add_argument("--only", choices=("all", "ops", "nearest"), default="all", help="run only the §8 rows or only the nearest join")
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
        if args.only == "nearest":
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


if __name__ == "__main__":
    main()
