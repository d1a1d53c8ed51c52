"""CPU restatement (oracle) of the host arithmetic around stage 2's two networks that the frame kernels of
csrc/stage2_io.cu reproduce: load_image + InputPadder.pad + cat, and cv2.resize(tensor2img(t)) + save_img
(src/models/utils.py), with OpenCV's bilinear resize written out in numpy (no cv2 call inside).

TEST INFRASTRUCTURE ONLY (see oracle/atlas_oracle.py): nothing in the product imports this module."""
import numpy as np

from . import loader_oracle as LO


# ----------------------------------------------------------------------------------------------------------------
# cv2.resize(INTER_LINEAR) in general — up-scaling too, any channel count, fp32 or float64 images — as the stage-2
# script meets it (src/models/utils.py: load_image resizes a float64 atlas frame up to the content's size, tensor2img's
# caller squeezes a padded fp32 tensor to the original size).  What up-scaling adds to the rules stated above
# resize_bilinear_down in oracle/loader_oracle.py (whose taps this shares):
#   * the horizontal pass zeroes the weight of a position outside [0, src - 1]; the VERTICAL pass does not — it only
#     clips the two row indices into the image, so a border row is R*(1-b) + R*b, which is not always R
#   * a float64 image keeps fp32 positions and weights; they are widened, and the products and sums are float64
#   * equal sizes are a copy
# This is OpenCV's own code path.  A build with Intel IPP hands 1-, 3- and 4-channel float images to IPP instead,
# whose results differ in the low bits (positions in float64) and are not restated: tests/test_stage2_resize_oracle.py
# pins these functions against cv2.resize with cv2.ipp.setUseIPP(False).  The exactly-half path of fp32 images with
# 1 or 4 channels is summed in another order by OpenCV's vector code and is refused here (nothing in the project
# meets it: flows have 2 channels, frames 3).
# ----------------------------------------------------------------------------------------------------------------
def _resize_linear(img, neww: int, newh: int, dt):
    img = np.asarray(img, dtype=dt)
    img = img[:, :, None] if img.ndim == 2 else img
    h, w, cn = img.shape
    if (h, w) == (newh, neww):
        return img.copy()
    c = lambda a: a.astype(dt)
    if h == 2 * newh and w == 2 * neww:
        assert dt is np.float64 or cn in (2, 3), "the fp32 half-size path is restated for 2 and 3 channels only"
        a, b, cc, d = img[0::2, 0::2], img[0::2, 1::2], img[1::2, 0::2], img[1::2, 1::2]
        return c(c(c(c(a + b) + cc) + d) * dt(0.25))
    sx, sx1, fx = LO._resize_taps(neww, w)
    scale = np.float64(h) / np.float64(newh)
    fy = ((np.arange(newh) + 0.5) * scale - 0.5).astype(np.float32)
    sy = np.floor(fy).astype(np.int64)
    fy = (fy - sy.astype(np.float32)).astype(np.float32)                   # weights kept, indices clipped
    sy, sy1 = np.clip(sy, 0, h - 1), np.clip(sy + 1, 0, h - 1)
    a0, a1 = c(np.float32(1) - fx)[None, :, None], c(fx)[None, :, None]
    b0, b1 = c(np.float32(1) - fy)[:, None, None], c(fy)[:, None, None]
    rows = c(c(img[:, sx] * a0) + c(img[:, sx1] * a1))
    return c(c(rows[sy] * b0) + c(rows[sy1] * b1))


def resize_linear_f32(img, neww: int, newh: int):
    """cv2.resize(img, (neww, newh), interpolation=cv2.INTER_LINEAR) for an fp32 image (H, W[, C]) -> (newh, neww, C)."""
    return _resize_linear(img, neww, newh, np.float32)


def resize_linear_f64(img, neww: int, newh: int):
    """The same for a float64 image (what load_image resizes)."""
    return _resize_linear(img, neww, newh, np.float64)


def stage2_pad(h: int, w: int):
    """InputPadder's (left, right, top, bottom) for an (h, w) image: up to multiples of 32, rows at the bottom."""
    ph, pw = -h % 32, -w % 32
    return pw // 2, pw - pw // 2, 0, ph


def stage2_pack_input(content_u8, atlas_u8):
    """cat(InputPadder.pad(load_image(content), load_image(atlas, size=content size))) from decoded 8-bit images
    (H, W) / (H, W, 3) / (H, W, 4): [1, 6, Hp, Wp] fp32."""
    def unit(a):
        a = np.asarray(a) / 255.
        return np.repeat(a[:, :, None], 3, axis=2) if a.ndim == 2 else a[..., :3]
    c, a = unit(content_u8), unit(atlas_u8)
    h, w = c.shape[:2]
    x = np.concatenate([c, resize_linear_f64(a, w, h)], axis=2).astype(np.float32)
    left, right, _, bottom = stage2_pad(h, w)
    return np.pad(x, ((0, bottom), (left, right), (0, 0)), mode="edge").transpose(2, 0, 1)[None]


def stage2_emit(t, w: int, h: int):
    """save_img's bytes for cv2.resize(tensor2img(t), (w, h)): t [1, 3, Hp, Wp] fp32 -> uint8 BGR (h, w, 3)."""
    img = resize_linear_f32(np.transpose(np.asarray(t, dtype=np.float32)[0], (1, 2, 0)), w, h)[:, :, ::-1]
    return np.clip(img * 255.0, 0, 255).astype(np.uint8)
