"""Runs every entry point of the points-in-polygons join on a fixed set of indexes and saves the outputs; a helper of
test_gpu_pip_regimes.py, not a test module.

The join's switches (GPL_PIP_LD_HINTS, GPL_PIP_RASTER_LOG2, GPL_PIP_RASTER_MCELLS, GPL_PIP_SLOTS_X100) are read once
per process, so each variant needs a fresh process: the test starts this script with the variant's environment and
compares what it wrote with the oracle.

    python tests/pip_variant_child.py OUTDIR

writes OUTDIR/<case>.npz (ids, counts, pair lists of every entry point) and OUTDIR/meta.json (per case: stats(), kernel
launches of query_counts, stream-kernel launches bracketed by kernel timing)."""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (ROOT, HERE):
    if p not in sys.path:
        sys.path.insert(0, p)


def null_mask(n):
    """validity of the Point column: nulls at rows 0, 127, 128, 129, n - 1 and every 5th row"""
    valid = np.ones(n, dtype=bool)
    valid[::5] = False
    valid[[0, 127, 128, 129, n - 1]] = False
    return valid


def _nested():
    from geopolars_b200 import GeoArrowArray, GeometryType, synth

    sq = lambda x, y, s: [(x, y), (x + s, y), (x + s, y + s), (x, y + s), (x, y)]
    shapes = [[sq(0, 0, 100)], [sq(10, 10, 50)], [sq(20, 20, 20)], [sq(25, 25, 5)], [sq(70, 70, 10), sq(72, 72, 3)]]
    xy, ro, go = synth.star_polygons(64, 8, cell=12.5)
    shapes += [[xy[ro[i]:ro[i + 1]].tolist()] for i in range(64)]
    return GeoArrowArray.from_shapes(GeometryType.POLYGON, shapes)


def cases():
    """name -> (polygon GeoArrowArray, points (n, 2)).  Deterministic: the test recomputes them for the oracle."""
    from geopolars_b200 import GeoArrowArray, GeometryType, synth
    from test_gpu_pip import _holes_and_multis
    from test_gpu_pip_regimes import field_points, star_field

    out = {}
    out["stars2500"] = star_field(2500, holes=False, seed=1)  # POLYGON rows without holes
    out["field2500"] = star_field(2500, holes=True, seed=2)
    out["multi2500"] = star_field(2500, holes=True, seed=2, multi=True)
    out["holes_multis"] = GeoArrowArray.from_shapes(GeometryType.MULTIPOLYGON, _holes_and_multis())
    out["nested"] = _nested()
    xy, ro, go = synth.star_polygons(16_900, 130)  # the largest case: 16 900 rows
    out["stars16900"] = GeoArrowArray.polygons(xy, ro, go)
    out["one"] = GeoArrowArray.from_shapes(GeometryType.POLYGON, [[[(0.0, 0.0), (4.0, 1.0), (5.0, 5.0), (1.0, 3.5), (0.0, 0.0)]]])
    # one million points on the 16 900 stars: several tiles per warp, so the walk queue carries points across tiles
    n_pts = {"stars16900": 1_000_000}
    return {k: (v, field_points(v, n_pts.get(k, 150_000), seed=len(k))) for k, v in out.items()}


def run(outdir):
    import torch

    from geopolars_b200 import GeoArrowArray
    from geopolars_b200.engine import Context, PipIndex

    ctx = Context(0)
    meta = {}
    for name, (polys, pts) in cases().items():
        idx = PipIndex(ctx.upload(polys))
        res = {}
        res["q_first"], res["q_cnt"] = idx.query(pts, with_count=True)
        res["q_only"] = idx.query(pts)
        before = ctx.launch_count
        res["c_first"], res["c_counts"] = idx.query_counts(pts)
        launches_counts = ctx.launch_count - before
        res["p_lhs"], res["p_rhs"] = idx.pairs(pts)
        d_arr = ctx.upload(GeoArrowArray.points(pts, valid=null_mask(len(pts))))
        res["a_first"], res["a_cnt"] = idx.query_array(d_arr, with_count=True)
        res["pa_lhs"], res["pa_rhs"] = idx.pairs_array(d_arr)
        d_pts = torch.from_numpy(pts).cuda()
        d_first = torch.empty(len(pts), dtype=torch.int32, device="cuda")
        d_cnt = torch.empty(len(pts), dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        idx.query_device(d_pts.data_ptr(), len(pts), d_first.data_ptr(), d_cnt.data_ptr())
        ctx.synchronize()
        res["d_first"], res["d_cnt"] = d_first.cpu().numpy(), d_cnt.cpu().numpy()
        ctx.kernel_timing(True)
        idx.query(pts)
        _, timed = ctx.kernel_timing_read()
        ctx.kernel_timing(False)
        np.savez(os.path.join(outdir, name + ".npz"), **res)
        meta[name] = {"stats": idx.stats(), "launches_counts": launches_counts, "timed_stream_launches": timed}
        idx.free()
        d_arr.free()
    ctx.synchronize()
    with open(os.path.join(outdir, "meta.json"), "w") as f:
        json.dump(meta, f)
    ctx.close()


if __name__ == "__main__":
    run(sys.argv[1])
