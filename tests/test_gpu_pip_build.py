"""The points-in-polygons index build writes the same tables it wrote when these digests were recorded.

For each case the test builds the index and compares the SHA-256 of four of its tables (the raster words, cand01, the cell
and part records, as `PipIndex.dump` returns them) and its `stats()` with digests pinned at commit 8b0dd1d.  They were
recorded on one H100 80GB HBM3 (700 W power limit) in the run where that commit's build with one thread per y-bucket and
a static deal of raster items produced the same bytes as its default build (DESIGN.md §4.2 "Build").  Every raster write is
an atomicOr of codes that compose in any order, so the bytes do not depend on how the build distributes its work.  The edge
lists (f64 records and FP32 lists) are left out: their order within a bucket comes from atomic cursors and differs from run
to run.

Cases: bench configs 2 and 4, the 151 k / 600 k / 2.2 M / 5 M star fields of test_gpu_pip_regimes.py (rs = 3, 2, 1, 1),
holes, MULTIPOLYGON rows and a degenerate axis.  The digests are of the default index geometry, so the test refuses to run
while one of the seams that change it is set in the environment."""
import hashlib
import os

import pytest

pytestmark = pytest.mark.gpu

SEAMS = ("GPL_PIP_RASTER_LOG2", "GPL_PIP_RASTER_MCELLS", "GPL_PIP_SLOTS_X100")
TABLES = ("raster", "cand01", "cells", "parts")
# case -> (stats(), SHA-256 of the tables in TABLES order)
PINNED = {
    "config2": ({"deferred": 0, "fine_cells_per_axis": 3200, "raster_log2": 5, "raster_walk_cells": 2339015,
         "raster_inside_cells": 2589952, "parts_not_fast": 0, "bytes": 68901120, "coarse_cells_per_axis": 100},
        ("14e66d69d4df48f4373f0df57324de99eebfe8741abad6b31bf6d2a6da700ce6", "7a304689b24a66af6f64315ce7f0c7605677bc170c1e1ccd932a2a73c7f3cf16",
         "1fd68338bb628020e7603eadd0804d79ce79a712f0ebeec48c7b06d97575d803", "49741328e45c96659850bdc6ef6efb4eeb9efca974fc7179639dbf58f9a5820e")),
    "config4": ({"deferred": 0, "fine_cells_per_axis": 4096, "raster_log2": 7, "raster_walk_cells": 1038881,
         "raster_inside_cells": 5446039, "parts_not_fast": 0, "bytes": 14766592, "coarse_cells_per_axis": 32},
        ("345580e2b4f20c5dfa9ce9cf03890a335718d826ca124244d7fb8ccfd93a8717", "f93e9a54acd7847c9ca2b633fb8a0d3907a69c377232056cd0cb614de9a245c7",
         "21c821c1c749ba6247f478a710d65c69b549d01c9702be48920d4d916fc01595", "57cdb6fe2ae4e9f3189487b134b6ee4d070ded02986d8b2626ed32f21efe302e")),
    "field151000": ({"deferred": 0, "fine_cells_per_axis": 3112, "raster_log2": 3, "raster_walk_cells": 6368352,
         "raster_inside_cells": 1159721, "parts_not_fast": 0, "bytes": 115204608, "coarse_cells_per_axis": 389},
        ("18dde3e630da4067ae13f484fe0d48652c8a48ff7ee6b03aa88f13d5a3a98814", "f423e9e27ff18e46e850d47a76469438b3749e0abc1ec5bef97c595ddfd65800",
         "5b851e6791eac01d8e1b686661584c507e0f8e94e9ec8f22bd35ed6036752268", "5a36d8e5d51bdb488e3a40353f3a45347495f6769d48bbc8e860d864b13b7ffe")),
    "field600000": ({"deferred": 0, "fine_cells_per_axis": 3100, "raster_log2": 2, "raster_walk_cells": 8021676,
         "raster_inside_cells": 646652, "parts_not_fast": 0, "bytes": 443566848, "coarse_cells_per_axis": 775},
        ("e8038901e4e90c580f293ff3c8810ade3d547807a2920f322f0f5787dcefe29f", "33125df5ebb9c0afc245c03fcfd15712e842c863159545e7cc4f3b661ebea0b7",
         "0c0e9427a760c13646678ffe54485c5d56ab5f8b93c2d6095114cd50b2fb6b72", "646a9207d1b857a62eb7037dd518bb1b43063cebdc38260b8d3f744acb416396")),
    "field2200000": ({"deferred": 0, "fine_cells_per_axis": 2968, "raster_log2": 1, "raster_walk_cells": 8601146,
         "raster_inside_cells": 48426, "parts_not_fast": 0, "bytes": 1613959680, "coarse_cells_per_axis": 1484},
        ("f30914b3a869d10517e9b40aed6cb881204a1ffab24145fb9c0df663274b4401", "4ac4cdf6966dec94ca4007fc5db8cdca7b4a9cb380823b495dda93cd43dcc8b0",
         "37b9e03f467b85ef84d90103aba5998ac4829748e4491031bb672e052d6b1809", "f68f33f7ba6a1e80667a44d0db278924e028ca22a92ed58ea9678769cb716454")),
    "field5000000": ({"deferred": 0, "fine_cells_per_axis": 4096, "raster_log2": 1, "raster_walk_cells": 16524693,
         "raster_inside_cells": 37699, "parts_not_fast": 0, "bytes": 3621481216, "coarse_cells_per_axis": 2048},
        ("04f96af1539bbe4b4eb77e1001a478e617a185ed60cff545a9506d572e017b83", "cd8c53b4e5a44c434b849b550b37b5ebef882260c3dcec3275cc65d8fc8e832d",
         "9a71ed2f6babd60ed0eeb9a10e631c6733cc581c5948807e0877f83961dc1503", "33b21f20c1b34394c53b4eafd01a7b7cc3991d3a2ff69e176fddb90523c9b5c1")),
    "field151000-holes": ({"deferred": 0, "fine_cells_per_axis": 3112, "raster_log2": 3, "raster_walk_cells": 6373153,
         "raster_inside_cells": 1154899, "parts_not_fast": 1697, "bytes": 120264704, "coarse_cells_per_axis": 389},
        ("9f4e9c7e764d4cdb08491f6bf6284478eace3c7d87b3e5c03cbc81e8af9a3ee6", "f423e9e27ff18e46e850d47a76469438b3749e0abc1ec5bef97c595ddfd65800",
         "b2c47215811895c0d534c0dd803d58f5550fae0a6b5abeec671f9095f66d9bec", "ddf465b63f06041f84bdbe617b191e92ecfbaf7025576c61435b5d83b7099509")),
    "field151000-multi": ({"deferred": 0, "fine_cells_per_axis": 3112, "raster_log2": 3, "raster_walk_cells": 6373153,
         "raster_inside_cells": 1154899, "parts_not_fast": 151000, "bytes": 68665600, "coarse_cells_per_axis": 389},
        ("9f4e9c7e764d4cdb08491f6bf6284478eace3c7d87b3e5c03cbc81e8af9a3ee6", "e50dba9d65c70b329702d567f4f210e4c43dd7ebcd6d1f90bdbd819765eac086",
         "4896311a5184d24a31529efd9c7d683e2784e1633fbf895612ab2599e85fe97b", "f7468c09f6ada2fec7e7b753cf31af0a9a01576e98def801750a4bf6ece77167")),
    "holes_multis": ({"deferred": 0, "fine_cells_per_axis": 256, "raster_log2": 7, "raster_walk_cells": 4418,
         "raster_inside_cells": 11268, "parts_not_fast": 4, "bytes": 36096, "coarse_cells_per_axis": 2},
        ("c13de328f2d20e377c80db7be5ec6c7fab1803e19778249ed23d0aa5c7bccb81", "17e74bbc23e3fc1c51a606335590fdb785938be40f2607256af7a096f8fecf10",
         "c9b4214737919cbb01628768ebd04ecfaee40844ab80f568228591d4d693541c", "dd93208504f6b0c600043092d4fed0b9d91e96c143f329d71c93b6596681922a")),
    "flat": ({"deferred": 0, "fine_cells_per_axis": 896, "raster_log2": 7, "raster_walk_cells": 802816,
         "raster_inside_cells": 0, "parts_not_fast": 0, "bytes": 418560, "coarse_cells_per_axis": 7},
        ("1daf888a838d40d6faa84423f92ec32836141d5f73821ad79a8b59bb3806eabd", "65baee4208dae5472dde2214267c7e0ea61a31a39f9463f0f3441002b1580316",
         "5f9db864b9f1de5fb82faaf19d516f52ab3dd38c474c605ba1447dbed4de56d7", "e98f95312cfa84afaf2140856ae062d95db8fd79a1d5d7eafb7112efeb291729")),
}
RASTER_LOG2 = {"config2": 5, "config4": 7, "field151000": 3, "field600000": 2, "field2200000": 1, "field5000000": 1}


def build_case(name):
    """the polygon GeoArrowArray of one case.  Deterministic."""
    from geopolars_b200 import GeoArrowArray, GeometryType, synth
    from test_gpu_pip import _holes_and_multis
    from test_gpu_pip_regimes import star_field

    if name == "config2":
        return GeoArrowArray.polygons(*synth.star_polygons(10_000, 100, 10.0, 64))
    if name == "config4":
        return GeoArrowArray.polygons(*synth.star_polygons(1_000, 32, 31.25, 64))
    if name.startswith("field"):
        P, _, form = name[len("field"):].partition("-")
        P = int(P)
        return star_field(P, holes=form != "", seed=P % 1000, multi=form == "multi")
    if name == "holes_multis":
        return GeoArrowArray.from_shapes(GeometryType.MULTIPOLYGON, _holes_and_multis())
    assert name == "flat"
    # every coordinate on one horizontal line: a degenerate y axis (the raster is all "walk")
    return GeoArrowArray.from_shapes(GeometryType.POLYGON,
                                     [[[(float(i), 2.0), (i + 3.0, 2.0), (i + 1.5, 2.0), (float(i), 2.0)]] for i in range(40)])


@pytest.mark.parametrize("case", list(PINNED))
def test_index_matches_pinned_build(ctx, case):
    from geopolars_b200.engine import PipIndex

    seams = [k for k in SEAMS if k in os.environ]
    assert not seams, f"unset {seams}: the pinned digests are of the default index geometry"
    d = ctx.upload(build_case(case))
    idx = PipIndex(d)
    try:
        st = idx.stats()
        got = {t: idx.dump(t) for t in TABLES}
    finally:
        idx.free()
        d.free()
    want_stats, want_sha = PINNED[case]
    assert st == want_stats, st
    if case in RASTER_LOG2:  # configs 2 and 4 and every field regime are reached
        assert st["raster_log2"] == RASTER_LOG2[case], st
    if case == "flat":  # degenerate axis: all "walk"
        assert st["raster_walk_cells"] == st["fine_cells_per_axis"] ** 2, st
    for t, h in zip(TABLES, want_sha):
        assert len(got[t]) > 0, t
        assert hashlib.sha256(got[t].tobytes()).hexdigest() == h, t
