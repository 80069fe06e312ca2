"""The points-in-polygons index comes out the same whichever way the build distributes its work.

The raster phase of the build claims (part, row-chunk) items from a global counter (DESIGN.md §4.2 "Build");
GPL_PIP_BUILD_LEGACY=1 restores the static deal of (part, 32-row) items.  Every raster write is an atomicOr of codes that
compose in any order, so both must produce the same index byte for byte: the raster words, cand01, the cell and part
records and stats().  The edge lists (f64 records and FP32 lists) are left out: their order within a bucket comes from
atomic cursors and differs from run to run on either path.

Cases (tests/pip_build_child.py): bench configs 2 and 4, the 151 k / 600 k / 2.2 M / 5 M star fields of
test_gpu_pip_regimes.py (rs = 3, 2, 1, 1), holes, MULTIPOLYGON rows and a degenerate axis.  Each build variant runs in a
child process, because the switches are read once per process."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
_SWITCHES = ("GPL_PIP_BUILD_LEGACY", "GPL_PIP_RASTER_LOG2", "GPL_PIP_RASTER_MCELLS", "GPL_PIP_SLOTS_X100")
VARIANTS = {
    "default": {},
    "legacy": {"GPL_PIP_BUILD_LEGACY": "1"},
}


def run_build(tmp_path_factory, name):
    out = tmp_path_factory.mktemp("pip-build-" + name)
    env = {k: v for k, v in os.environ.items() if k not in _SWITCHES}
    env.update(VARIANTS[name])
    subprocess.run([sys.executable, os.path.join(HERE, "pip_build_child.py"), str(out)], env=env, timeout=900, check=True)
    with open(out / "meta.json") as f:
        meta = json.load(f)
    return {k: dict(np.load(out / f"{k}.npz")) for k in meta}, meta


@pytest.fixture(scope="module")
def legacy(tmp_path_factory):
    return run_build(tmp_path_factory, "legacy")


@pytest.mark.parametrize("variant", ["default"])
def test_index_identical_to_legacy_build(variant, legacy, tmp_path_factory):
    tables, meta = run_build(tmp_path_factory, variant)
    want_tables, want_meta = legacy
    assert sorted(meta) == sorted(want_meta)
    regimes = {(m["raster_log2"], m["coarse_cells_per_axis"]) for m in meta.values()}
    assert {5, 7, 3, 2, 1} <= {rs for rs, _ in regimes}, regimes  # configs 2 and 4 and every field regime were reached
    assert meta["flat"]["raster_walk_cells"] == meta["flat"]["fine_cells_per_axis"] ** 2  # degenerate axis: all "walk"
    for case in meta:
        assert meta[case] == want_meta[case], case
        for t, v in want_tables[case].items():
            assert len(v) > 0, (case, t)
            assert np.array_equal(tables[case][t], v), (case, t, np.nonzero(tables[case][t] != v)[0][:8])
