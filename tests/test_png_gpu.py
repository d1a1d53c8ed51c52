"""b200_png_encode (csrc/png_encode.cu) against the installed OpenCV's level-0 PNG writer, byte for byte, at the shapes
stage 2 writes and at the edges of the layout (small-window zlib headers, rows split across stored blocks), and
Stage2.frame_png against cv2.imencode of Stage2.frame's images."""
import types

import cv2
import numpy as np
import pytest
import torch

import png_oracle as O
from b200 import _native as N
from b200 import nn as K
from b200 import png as P
from b200 import stage2 as S2

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SHAPES = [(1, 1), (17, 5), (1, 22000), (5, 21846), (270, 1440), (1080, 1920), (1080, 5760)]


def _cv2(img):
    ok, buf = cv2.imencode(".png", img, [cv2.IMWRITE_PNG_COMPRESSION, 0])
    assert ok
    return buf.tobytes()


def _encode(img):
    """(file bytes, the filter byte of each row as the filter kernel wrote it)."""
    h, w = img.shape[:2]
    plan = P.plan(h, w, DEV)
    ws = torch.full((plan.workspace_bytes,), 0xA5, dtype=torch.uint8, device=DEV)
    out = torch.full((plan.file_bytes + 64,), 0xA5, dtype=torch.uint8, device=DEV)
    got = P.encode(torch.from_numpy(img).to(DEV), out=out, workspace=ws)
    assert got.data_ptr() == out.data_ptr() and got.numel() == plan.file_bytes
    assert (out[plan.file_bytes:] == 0xA5).all(), "bytes past the file were written"
    filters = ws[:h * (3 * w + 1)].view(h, 3 * w + 1)[:, 0].cpu().numpy()
    return got.cpu().numpy().tobytes(), filters


@pytest.mark.parametrize("h,w", SHAPES, ids=lambda v: str(v))
def test_device_file_equals_opencv(h, w):
    for kind in O.KINDS:
        img = O.content(kind, h, w)
        got, filters = _encode(img)
        want_filters = O.filter_rows(img)[0]
        bad = np.flatnonzero(filters != want_filters)
        assert bad.size == 0, "%s: row %d takes filter %d, libpng's choice is %d (%d rows differ)" % (
            kind, bad[0], filters[bad[0]], want_filters[bad[0]], bad.size)
        want = _cv2(img)
        if got != want:
            i = next(k for k in range(min(len(got), len(want))) if got[k] != want[k]) if len(got) == len(want) else -1
            pytest.fail("%s: %d bytes against %d, first difference at byte %d" % (kind, len(got), len(want), i))


def test_graph_replay_gives_the_same_bytes():
    h, w = 270, 1440
    imgs = [torch.from_numpy(O.content(k, h, w)).to(DEV) for k in ("random", "gradient")]
    plan = P.plan(h, w, DEV)
    ws = torch.empty(plan.workspace_bytes, dtype=torch.uint8, device=DEV)
    out = torch.empty(plan.file_bytes, dtype=torch.uint8, device=DEV)
    src = torch.empty_like(imgs[0])
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            P.encode(src, out=out, workspace=ws)
    for img in imgs + imgs[:1]:
        src.copy_(img)
        out.zero_()
        g.replay()
        torch.cuda.synchronize()
        assert out.cpu().numpy().tobytes() == _cv2(img.cpu().numpy())


def test_arguments_are_reported_not_overrun():
    img = torch.from_numpy(O.content("random", 17, 5)).to(DEV)
    plan = P.plan(17, 5, DEV)
    with pytest.raises(N.B200Error, match="output capacity"):
        P.encode(img, out=torch.empty(plan.file_bytes - 1, dtype=torch.uint8, device=DEV))
    with pytest.raises(N.B200Error, match="workspace"):
        P.encode(img, workspace=torch.empty(plan.workspace_bytes - 1, dtype=torch.uint8, device=DEV))
    with pytest.raises(N.B200Error, match="contiguous uint8"):
        P.encode(img.float())
    with pytest.raises(N.B200Error, match="contiguous uint8"):
        P.encode(torch.zeros(17, 10, 3, dtype=torch.uint8, device=DEV)[:, ::2])
    with pytest.raises(N.B200Error, match="contiguous uint8"):
        P.encode(torch.zeros(17, 5, 4, dtype=torch.uint8, device=DEV))
    assert _encode(O.content("random", 17, 5))[0] == _cv2(O.content("random", 17, 5))      # and the library still works


def test_frame_png_equals_opencv_of_frame():
    K.set_conv_precision("tc" if N.lib().b200_device_supports_tc() else "fp32")
    from src.models.network_filter import UNet
    from src.models.network_local import TransformNet
    torch.manual_seed(5)
    unet = UNet(in_channels=6, out_channels=3, init_features=32).to(DEV).eval()
    tn = TransformNet(types.SimpleNamespace(nf=32, norm="IN", model="TransformNet", blocks=5), nc_in=12, nc_out=3)
    tn = tn.to(DEV).eval()
    rng = np.random.default_rng(3)
    frames = [(rng.integers(0, 256, (67, 101, 3), dtype=np.uint8), rng.integers(0, 256, (23, 37, 3), dtype=np.uint8))
              for _ in range(3)]
    a, b = S2.Stage2(unet, tn, DEV), S2.Stage2(unet, tn, DEV)
    held = None
    for i, (c, s) in enumerate(frames):
        imgs = {k: v.copy() for k, v in a.frame(c, s).items()}
        files = b.frame_png(c, s)
        assert set(files) == {"concat", "filter", "final"}
        for k in files:
            assert files[k].dtype == np.uint8 and files[k].tobytes() == _cv2(imgs[k]), (i, k)
        if i == 0:
            held = {k: (v, v.tobytes()) for k, v in files.items()}
        if i == 1:                                 # frame 0's files are still valid after one more call
            assert all(v.tobytes() == want for v, want in held.values())
