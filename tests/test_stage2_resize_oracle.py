"""oracle/stage2_io_oracle.py's general bilinear resize (resize_linear_f64 / resize_linear_f32) pinned bit for bit against
cv2.resize itself, on the CPU: the arithmetic the stage-2 frame kernels (csrc/stage2_io.cu) restate, so their bit-exact
claim can be checked on a machine whose OpenCV build differs.

cv2.resize is called with OpenCV's IPP back end switched off: a build with Intel IPP hands 1-, 3- and 4-channel float
images to IPP, whose results differ from OpenCV's own code in the low bits; what is restated is OpenCV's own code."""
import cv2
import numpy as np
import pytest

from oracle import loader_oracle
from oracle import stage2_io_oracle as LO


@pytest.fixture(autouse=True)
def _opencv_own_code():
    was = cv2.ipp.useIPP()
    cv2.ipp.setUseIPP(False)
    yield
    cv2.ipp.setUseIPP(was)


# (source h, w) -> (destination h, w)
SIZES = [((120, 213), (480, 852)),          # x4
         ((120, 213), (480, 854)),          # x4 rows, x4.009 columns
         ((270, 480), (1080, 1920)),
         ((1088, 1920), (1080, 1920)),      # x0.9926 rows, equal columns
         ((64, 96), (64, 96)),              # equal: a copy
         ((1, 1), (7, 9)), ((1, 5), (4, 5)), ((5, 1), (5, 4)), ((7, 9), (1, 1)),
         ((67, 101), (23, 37)), ((23, 37), (67, 101)),
         ((64, 96), (32, 48)),              # exactly half in both dimensions: the 2x2 mean
         ((32, 40), (16, 23)), ((32, 40), (16, 40))]   # half in one dimension only: bilinear


def _cv(img, dw, dh):
    out = cv2.resize(img[:, :, 0] if img.shape[2] == 1 else img, (dw, dh), interpolation=cv2.INTER_LINEAR)
    return out.reshape(dh, dw, img.shape[2])


@pytest.mark.parametrize("cn", [1, 3, 4], ids=["grey", "rgb", "rgba"])
@pytest.mark.parametrize("src,dst", SIZES, ids=lambda s: "%dx%d" % s)
def test_f64_resize_equals_opencv(src, dst, cn):
    rng = np.random.default_rng(src[0] * 7 + dst[1] + cn)
    img = rng.integers(0, 256, (*src, cn)) / 255.                     # what load_image resizes
    got = LO.resize_linear_f64(img, dst[1], dst[0])
    assert got.dtype == np.float64 and np.array_equal(got, _cv(img, dst[1], dst[0]))


@pytest.mark.parametrize("cn", [2, 3], ids=["flow", "rgb"])
@pytest.mark.parametrize("src,dst", SIZES, ids=lambda s: "%dx%d" % s)
def test_f32_resize_equals_opencv(src, dst, cn):
    rng = np.random.default_rng(src[1] * 5 + dst[0] + cn)
    img = (rng.random((*src, cn)) * 1.4 - 0.2).astype(np.float32)     # a network output, a little outside [0, 1]
    got = LO.resize_linear_f32(img, dst[1], dst[0])
    assert got.dtype == np.float32 and np.array_equal(got, _cv(img, dst[1], dst[0]))


def test_up_scaled_border_rows_are_weighted_not_copied():
    """The vertical pass clips row indices but keeps its weights: R*(1-b) + R*b in the first row of a x4 up-scale is
    not R for every R, while the first column (weight zeroed by the horizontal pass) is a copy."""
    rng = np.random.default_rng(3)
    img = rng.integers(0, 256, (30, 40, 3)) / 255.
    out = LO.resize_linear_f64(img, 160, 120)
    assert np.array_equal(out, _cv(img, 160, 120))
    assert np.array_equal(out[2:-2:4, 0], _cv(img, 160, 120)[2:-2:4, 0])
    assert not np.array_equal(out[0, ::4], LO.resize_linear_f64(img[:1], 160, 1)[0, ::4])


def test_general_resize_agrees_with_the_flow_resize_where_that_is_defined():
    rng = np.random.default_rng(4)
    flow = rng.standard_normal((48, 64, 2)).astype(np.float32)
    for w, h in ((40, 30), (32, 24), (64, 48), (64, 31)):
        assert np.array_equal(loader_oracle.resize_bilinear_down(flow, w, h), LO.resize_linear_f32(flow, w, h)), (w, h)


def test_half_size_fp32_is_refused_for_channel_counts_opencv_vectorises():
    with pytest.raises(AssertionError):
        LO.resize_linear_f32(np.zeros((8, 8, 4), np.float32), 4, 4)
