"""Host side of the stage-2 frame path, no GPU: b200.stage2's padding geometry is InputPadder's, the numpy statement of
the two frame kernels (oracle/stage2_io_oracle.py stage2_pack_input / stage2_emit) equals the helpers of
src/models/utils.py bit for bit (OpenCV running its own resize code, see tests/test_stage2_resize_oracle.py), and the
script still parses the reference's command line."""
import importlib.util
import os

import cv2
import numpy as np
import pytest
import torch
from PIL import Image

from b200 import stage2 as S2
from oracle import stage2_io_oracle as LO
from src.models import utils as U

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(autouse=True)
def _opencv_own_code():
    was = cv2.ipp.useIPP()
    cv2.ipp.setUseIPP(False)
    yield
    cv2.ipp.setUseIPP(was)


def test_padding_geometry_is_the_padders(golden_dir):
    z = np.load(os.path.join(golden_dir, "stage2_io.npz"))
    sizes = [tuple(int(v) for v in k[4:].split("x")) for k in z.files if k.startswith("pad_")]
    assert sizes
    for h, w in sizes + [(1080, 1920), (480, 854), (67, 101), (64, 96), (1, 1), (32, 33)]:
        want = U.InputPadder((1, 3, h, w))._pad
        assert list(S2.pad_geometry(h, w)) == list(want) == list(LO.stage2_pad(h, w)), (h, w)
    for k in (k for k in z.files if k.startswith("pad_")):
        assert list(S2.pad_geometry(*(int(v) for v in k[4:].split("x")))) == list(z[k])


# content (h, w, channels or 0 for a 2-D grey image), atlas frame likewise
GEOMETRIES = [((64, 96, 3), (64, 96, 3)), ((480, 854, 3), (120, 213, 3)), ((67, 101, 3), (23, 37, 3)),
              ((67, 101, 0), (23, 37, 3)), ((67, 101, 3), (23, 37, 4)), ((48, 80, 3), (67, 101, 3)),
              ((48, 80, 3), (96, 160, 0))]


def _u8(rng, shape):
    return rng.integers(0, 256, shape[:2] + ((shape[2],) if shape[2] else ()), dtype=np.uint8)


@pytest.mark.parametrize("content,atlas", GEOMETRIES, ids=lambda s: "%dx%dx%d" % s)
def test_pack_oracle_equals_the_host_helpers(content, atlas, tmp_path):
    rng = np.random.default_rng(content[0] + atlas[1])
    c, a = _u8(rng, content), _u8(rng, atlas)
    Image.fromarray(c).save(str(tmp_path / "c.png"))
    Image.fromarray(a).save(str(tmp_path / "a.png"))
    ct, org = U.load_image(str(tmp_path / "c.png"), device="cpu", resize=False)
    at, _ = U.load_image(str(tmp_path / "a.png"), size=org, device="cpu", resize=False)
    want = torch.cat(U.InputPadder(ct.shape).pad(ct, at), dim=1).numpy()
    got = LO.stage2_pack_input(c, a)
    assert got.dtype == np.float32 and got.shape == want.shape and np.array_equal(got, want)
    assert np.array_equal(S2.host_input(c, a, "cpu").numpy(), want)


@pytest.mark.parametrize("h,w", [(64, 96), (480, 854), (67, 101), (16, 16)], ids=lambda v: str(v))
def test_emit_oracle_equals_save_img(h, w, tmp_path):
    left, right, _, bottom = S2.pad_geometry(h, w)
    rng = np.random.default_rng(h)
    t = (rng.random((1, 3, h + bottom, w + left + right)) * 1.4 - 0.2).astype(np.float32)
    t[0, :, ::3, ::5] = (rng.integers(-20, 280, t[0, :, ::3, ::5].shape) / 255.0).astype(np.float32)
    U.save_img(cv2.resize(U.tensor2img(torch.from_numpy(t)), (w, h), cv2.INTER_LINEAR), str(tmp_path / "o.png"))
    want = cv2.imread(str(tmp_path / "o.png"), cv2.IMREAD_UNCHANGED)
    got = LO.stage2_emit(t, w, h)
    assert np.array_equal(got, want) and got.min() == 0 and got.max() == 255


def test_script_parses_the_reference_command_line():
    path = os.path.join(ROOT, "all-in-one-deflicker_b200", "src", "neural_filter_and_refinement.py")
    spec = importlib.util.spec_from_file_location("stage2_script", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    o = mod.parser.parse_args(["--video_name", "clip", "--fps", "10", "--gpu", "0", "--ckpt_filter", "f.pth", "--ckpt_local",
                               "l.pth"])
    assert (o.video_name, o.fps, o.gpu, o.ckpt_filter, o.ckpt_local, o.sync_io) == ("clip", 10, 0, "f.pth", "l.pth", False)
    assert mod.parser.parse_args(["--video_name", "clip", "--sync_io"]).sync_io
