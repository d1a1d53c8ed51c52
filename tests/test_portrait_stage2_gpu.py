"""Stage 2 on PORTRAIT frames (height the larger side): the filter-input packing and 8-bit emission of test_stage2_io_gpu
and the launch-by-launch UNet / TransformNet checks of test_net_launches_gpu, at the portrait counterparts of their
landscape geometries.  Every landscape case there has H < W; here InputPadder pads a frame whose height is the larger
side (and, in one case, only its width), and the networks' halos, stride-2 phases and the TransformNet state take
that shape.  Needs a GPU; same bounds as the files the checks come from."""
import pytest

import test_net_launches_gpu as TNL
import test_stage2_io_gpu as TIO
from b200 import nn as K
from b200 import stage2 as S2
from csrc_build import ensure_built
from test_stage2_io_gpu import _opencv_own_code  # noqa: F401  (autouse fixture: OpenCV's own arithmetic)

pytestmark = pytest.mark.gpu

# content (h, w, channels), atlas frame likewise
GEOMETRIES = [((854, 480, 3), (213, 120, 3)),        # 854 x 480 portrait, atlas frames at a quarter
              ((101, 67, 3), (37, 23, 3)),           # odd everything, both pads non-zero
              ((101, 67, 0), (37, 23, 3)),           # grey content
              ((128, 67, 3), (32, 17, 3))]           # height a multiple of 32: InputPadder pads the width only


def test_geometries_are_portrait_and_one_pads_only_the_width():
    for (h, w, _), (ah, aw, _) in GEOMETRIES:
        assert h > w and ah > aw
    left, right, _, bottom = S2.pad_geometry(128, 67)
    assert bottom == 0 and left + right == 29
    assert all(v > 0 for v in S2.pad_geometry(101, 67)[1::2]) and S2.pad_geometry(854, 480)[3] > 0


@pytest.mark.parametrize("content,atlas", GEOMETRIES, ids=lambda s: "%dx%dx%d" % s)
def test_pack_input_portrait(content, atlas, tmp_path):
    TIO.test_pack_input_equals_host_helpers_and_oracle(content, atlas, tmp_path)


@pytest.mark.parametrize("h,w", [(854, 480), (101, 67), (128, 67)], ids=lambda v: str(v))
def test_emit_portrait(h, w, tmp_path):
    TIO.test_emit_equals_save_img_inside_a_panel(h, w, tmp_path)


@pytest.mark.parametrize("precision", ["tc", "fp32"])
def test_networks_launch_by_launch_portrait(golden_dir, precision, monkeypatch):
    """The UNet on one 854 x 480 frame and the TransformNet on three (zero state, then two carried states)."""
    ensure_built()
    monkeypatch.setattr(TNL, "GEOMETRIES", [(854, 480)])
    prev = K.set_conv_precision(precision)
    try:
        TNL.test_stage2_networks_launch_by_launch(golden_dir, precision)
    finally:
        K.set_conv_precision(prev)
