"""Builds the points-in-polygons index of a fixed set of polygon columns and saves its tables; a helper of
test_gpu_pip_build.py, not a test module.

The build's switch GPL_PIP_BUILD_LEGACY is read once per process, so each variant of the build
runs in a fresh process: the test starts this script with the variant's environment and compares what it wrote.

    python tests/pip_build_child.py OUTDIR

writes OUTDIR/<case>.npz (the raster words, cand01, cell and part records as raw bytes) and OUTDIR/meta.json (per case:
stats() of the fresh index)."""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (ROOT, HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

TABLES = ("raster", "cand01", "cells", "parts")


def cases():
    """name -> polygon GeoArrowArray.  Deterministic."""
    from geopolars_b200 import GeoArrowArray, GeometryType, synth
    from test_gpu_pip import _holes_and_multis
    from test_gpu_pip_regimes import star_field

    out = {}
    xy, ro, go = synth.star_polygons(10_000, 100, 10.0, 64)  # bench config 2: rs = 5
    out["config2"] = GeoArrowArray.polygons(xy, ro, go)
    xy, ro, go = synth.star_polygons(1_000, 32, 31.25, 64)  # bench config 4: rs = 7
    out["config4"] = GeoArrowArray.polygons(xy, ro, go)
    for P in (151_000, 600_000, 2_200_000, 5_000_000):  # rs = 3, 2, 1, 1 (G capped at 2048)
        out[f"field{P}"] = star_field(P, holes=False, seed=P % 1000)
    out["field151000-holes"] = star_field(151_000, holes=True, seed=151_000 % 1000)
    out["field151000-multi"] = star_field(151_000, holes=True, seed=151_000 % 1000, multi=True)
    out["holes_multis"] = GeoArrowArray.from_shapes(GeometryType.MULTIPOLYGON, _holes_and_multis())
    # every coordinate on one horizontal line: a degenerate y axis (the raster is all "walk")
    flat = [[[(float(i), 2.0), (i + 3.0, 2.0), (i + 1.5, 2.0), (float(i), 2.0)]] for i in range(40)]
    out["flat"] = GeoArrowArray.from_shapes(GeometryType.POLYGON, flat)
    return out


def main(out_dir):
    from geopolars_b200.engine import Context, PipIndex

    ctx = Context(0)
    meta = {}
    for name, polys in cases().items():
        d = ctx.upload(polys)
        idx = PipIndex(d)
        np.savez(os.path.join(out_dir, f"{name}.npz"), **{t: idx.dump(t) for t in TABLES})
        meta[name] = idx.stats()
        idx.free()
        d.free()
    ctx.synchronize()
    with open(os.path.join(out_dir, "meta.json"), "w") as f:
        json.dump(meta, f)


if __name__ == "__main__":
    main(sys.argv[1])
