"""The points-in-polygons join refuses a device point column that is not 16-byte aligned (gpl_contains_join with
GPL_DEVICE): the stream kernel (k_pip_stream, geopolars_b200/csrc/k_pip.cu) reads each point as one 16-byte load, so such a
column is rejected on the host, before any launch, and the id column is left as it was."""
import pytest

from geopolars_b200 import GeoArrowArray, synth
from geopolars_b200._lib import GeopolarsError

pytestmark = pytest.mark.gpu


def test_misaligned_point_column_is_refused(ctx):
    import torch

    from geopolars_b200.engine import PipIndex

    xy, ro, go = synth.star_polygons(100, 10)
    idx = PipIndex(ctx.upload(GeoArrowArray.polygons(xy, ro, go)))
    d_pts = torch.from_numpy(synth.uniform_points(1_001, scale=100.0)).cuda()
    d_ids = torch.full((1_000,), -7, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    with pytest.raises(GeopolarsError, match="16-byte aligned") as e:
        idx.query_device(d_pts.data_ptr() + 8, 1_000, d_ids.data_ptr())  # x of row 0 is skipped: every point straddles
    assert e.value.code == -7  # GPL_ERR_INVALID_ARG
    ctx.synchronize()
    assert (d_ids.cpu().numpy() == -7).all()
    idx.query_device(d_pts.data_ptr() + 16, 1_000, d_ids.data_ptr())  # the same allocation one whole row in is accepted
    ctx.synchronize()
    assert (d_ids.cpu().numpy() != -7).all()
