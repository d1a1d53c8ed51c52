"""The stage-2 frame kernels (csrc/stage2_io.cu), b200.stage2.Stage2 and the script's frame loop against the host
arithmetic of src/models/utils.py they replace: every comparison is bit for bit.  The host side runs OpenCV's own resize
code (IPP switched off, see tests/test_stage2_resize_oracle.py), which is what the kernels restate."""
import importlib.util
import os
import types

import cv2
import numpy as np
import pytest
import torch
from PIL import Image

from b200 import _native as N
from b200 import nn as K
from b200 import stage2 as S2
from oracle import stage2_io_oracle as LO
from src.models import utils as U

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda:0"


@pytest.fixture(autouse=True)
def _opencv_own_code():
    was = cv2.ipp.useIPP()
    cv2.ipp.setUseIPP(False)
    yield
    cv2.ipp.setUseIPP(was)


def _u8(rng, shape):
    return rng.integers(0, 256, shape[:2] + ((shape[2],) if shape[2] else ()), dtype=np.uint8)


def _host_input(c_path, a_path, device):
    content, org = U.load_image(c_path, device=device, resize=False)
    style, _ = U.load_image(a_path, size=org, device=device, resize=False)
    return torch.cat(U.InputPadder(content.shape).pad(content, style), dim=1), org


# content (h, w, channels or 0 for a 2-D grey image), atlas frame likewise
GEOMETRIES = [((64, 96, 3), (64, 96, 3)),            # equal sizes: the copy path, no padding
              ((480, 854, 3), (120, 213, 3)),        # x4 / x4.009 up-scale, 10 columns of padding split 5 / 5, none below
              ((67, 101, 3), (23, 37, 3)),           # odd everything, both pads non-zero
              ((67, 101, 0), (23, 37, 3)),           # grey content
              ((67, 101, 3), (23, 37, 4)),           # RGBA atlas frame
              ((48, 80, 3), (67, 101, 3)),           # atlas frame larger than the content: down-scale
              ((48, 80, 3), (96, 160, 0))]           # exactly twice the content: the 2x2 mean


@pytest.mark.parametrize("content,atlas", GEOMETRIES, ids=lambda s: "%dx%dx%d" % s)
def test_pack_input_equals_host_helpers_and_oracle(content, atlas, tmp_path):
    rng = np.random.default_rng(content[0] + atlas[1])
    c, a = _u8(rng, content), _u8(rng, atlas)
    Image.fromarray(c).save(str(tmp_path / "c.png"))
    Image.fromarray(a).save(str(tmp_path / "a.png"))
    want, _ = _host_input(str(tmp_path / "c.png"), str(tmp_path / "a.png"), DEV)
    before = N.lib().b200_launch_count()
    got = S2.pack_input(torch.from_numpy(c).to(DEV), torch.from_numpy(a).to(DEV))
    assert N.lib().b200_launch_count() == before + 1
    assert got.shape == want.shape and got.shape[2] % 32 == 0 and got.shape[3] % 32 == 0
    assert torch.equal(got, want)
    assert np.array_equal(got.cpu().numpy(), LO.stage2_pack_input(c, a))


@pytest.mark.parametrize("h,w", [(64, 96), (480, 854), (67, 101), (16, 16)], ids=lambda v: str(v))
def test_emit_equals_save_img_inside_a_panel(h, w, tmp_path):
    left, right, _, bottom = S2.pad_geometry(h, w)
    rng = np.random.default_rng(h)
    t = (rng.random((1, 5, h + bottom, w + left + right)) * 1.4 - 0.2).astype(np.float32)      # both clamps are hit
    t[0, :, ::3, ::5] = (rng.integers(-20, 280, t[0, :, ::3, ::5].shape) / 255.0).astype(np.float32)
    sl = t[:, 1:4]                                                                             # a channel slice
    U.save_img(cv2.resize(U.tensor2img(torch.from_numpy(sl)), (w, h), cv2.INTER_LINEAR), str(tmp_path / "o.png"))
    want = cv2.imread(str(tmp_path / "o.png"), cv2.IMREAD_UNCHANGED)
    assert np.array_equal(want, LO.stage2_emit(sl, w, h)) and want.min() == 0 and want.max() == 255
    out = torch.full((h, 3 * w, 3), 0xA5, dtype=torch.uint8, device=DEV)
    S2.emit(torch.from_numpy(t).to(DEV)[:, 1:4], out, w, w)
    out = out.cpu().numpy()
    assert np.array_equal(out[:, w:2 * w], want)
    assert (out[:, :w] == 0xA5).all() and (out[:, 2 * w:] == 0xA5).all()


def test_entry_points_validate_and_are_graph_capturable():
    c = torch.zeros(40, 50, 3, dtype=torch.uint8, device=DEV)
    with pytest.raises(N.B200Error, match="multiples of 32"):
        S2.pack_input(c, c, out=torch.empty(1, 6, 40, 64, device=DEV))
    with pytest.raises(N.B200Error, match="1, 3 or 4 channels"):
        S2.pack_input(torch.zeros(40, 50, 2, dtype=torch.uint8, device=DEV), c)
    with pytest.raises(N.B200Error):
        S2.emit(torch.zeros(1, 3, 64, 64, device=DEV), torch.zeros(40, 50, 3, dtype=torch.uint8, device=DEV), 10, 50)
    rng = np.random.default_rng(0)
    c = torch.from_numpy(_u8(rng, (40, 50, 3))).to(DEV)
    a = torch.from_numpy(_u8(rng, (10, 13, 3))).to(DEV)
    x6, img = torch.empty(1, 6, 64, 64, device=DEV), torch.zeros(40, 50, 3, dtype=torch.uint8, device=DEV)
    want_x6 = S2.pack_input(c, a)
    want_img = torch.zeros_like(img)
    S2.emit(want_x6[:, 3:6], want_img, 0, 50)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            S2.pack_input(c, a, out=x6)
            S2.emit(x6[:, 3:6], img, 0, 50)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(x6, want_x6) and torch.equal(img, want_img)


# ---- the whole loop -------------------------------------------------------------------------------------------------
def _script():
    path = os.path.join(ROOT, "all-in-one-deflicker_b200", "src", "neural_filter_and_refinement.py")
    spec = importlib.util.spec_from_file_location("stage2_script", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _nets():
    from src.models.network_filter import UNet
    from src.models.network_local import TransformNet
    torch.manual_seed(5)
    unet = UNet(in_channels=6, out_channels=3, init_features=32).to(DEV).eval()
    tn = TransformNet(types.SimpleNamespace(nf=32, norm="IN", model="TransformNet", blocks=5), nc_in=12, nc_out=3)
    return unet, tn.to(DEV).eval()


def _host_loop(filter_net, local_net, content_names, style_names, dirs):
    """The frame loop on the host helpers of src/models/utils.py, as the reference's script has it."""
    frame_o1 = frame_p1 = None
    for i in range(len(content_names)):
        x6, org = _host_input(content_names[i], style_names[i], DEV)
        pred = filter_net(x6)
        if i == 0:
            frame_o2 = frame_o1 = frame_p1 = pred
        else:
            out, _ = local_net(torch.cat((pred, frame_o1, pred, frame_p1), dim=1), None)
            frame_o2 = pred + out
            frame_p1, frame_o1 = pred, frame_o2
        imgs = [cv2.resize(U.tensor2img(t), org, cv2.INTER_LINEAR) for t in (x6[:, 0:3], x6[:, 3:6], pred)]
        U.save_img(np.concatenate(imgs, axis=1), "{}/{:05d}.png".format(dirs["concat"], i))
        U.save_img(imgs[2], "{}/{:05d}.png".format(dirs["filter"], i))
        U.save_img(cv2.resize(U.tensor2img(frame_o2), org, cv2.INTER_LINEAR), "{}/{:05d}.png".format(dirs["final"], i))


def _dirs(root):
    d = {k: os.path.join(str(root), k) for k in ("concat", "filter", "final")}
    for v in d.values():
        os.makedirs(v)
    return d


def _files(dirs, n):
    out = {}
    for k, v in dirs.items():
        assert sorted(os.listdir(v)) == ["%05d.png" % i for i in range(n)]
        out[k] = [open(os.path.join(v, f), "rb").read() for f in sorted(os.listdir(v))]
    return out


def _sequence(folder, n, content, atlas, dtype=np.uint8):
    rng = np.random.default_rng(11)
    os.makedirs(os.path.join(folder, "content"))
    os.makedirs(os.path.join(folder, "atlas"))
    base = rng.integers(0, 256, atlas + (3,)).astype(np.float32)
    cn, an = [], []
    for i in range(n):
        a = np.clip(base + rng.normal(0, 4, base.shape), 0, 255).astype(np.uint8)
        c = cv2.resize(a, (content[1], content[0]), interpolation=cv2.INTER_CUBIC)
        c = np.clip(c * (0.8 + 0.4 * rng.random()) + rng.normal(0, 3, c.shape), 0, 255).astype(np.uint8)      # flicker
        cn.append(os.path.join(folder, "content", "%05d.png" % i))
        an.append(os.path.join(folder, "atlas", "%05d.png" % i))
        if dtype == np.uint16:
            cv2.imwrite(cn[-1], c[:, :, 1].astype(np.uint16))                 # 16-bit grey, samples in the 8-bit range
        else:
            Image.fromarray(c).save(cn[-1])
        Image.fromarray(a).save(an[-1])
    return cn, an


@pytest.mark.parametrize("precision", ["tc", "fp32"])
def test_loop_writes_the_same_files_as_the_host_loop(precision, tmp_path):
    if precision == "tc" and not N.lib().b200_device_supports_tc():
        pytest.skip("no tensor-core path on this device")
    K.set_conv_precision(precision)
    try:
        script = _script()
        unet, tn = _nets()
        cn, an = _sequence(str(tmp_path / "in"), 5, (270, 480), (68, 120))
        with torch.no_grad():
            host = _dirs(tmp_path / "host")
            _host_loop(unet, tn, cn, an, host)
            want = _files(host, 5)
            st = S2.Stage2(unet, tn, DEV)
            before = N.lib().b200_launch_count()
            for tag, sync_io in (("sync", True), ("piped", False), ("again", False)):
                d = _dirs(tmp_path / tag)
                script.run_frames(st, cn, an, d, sync_io=sync_io)          # run_frames resets the recurrence
                assert _files(d, 5) == want, tag
            assert N.lib().b200_launch_count() > before
        assert want["final"][1] != want["filter"][1]                           # the refinement did something
        img = cv2.imread(os.path.join(host["concat"], "00003.png"), cv2.IMREAD_UNCHANGED)
        assert img.shape == (270, 3 * 480, 3) and img.std() > 5
    finally:
        K.set_conv_precision("tc")


def test_reset_and_result_lifetime():
    K.set_conv_precision("tc" if N.lib().b200_device_supports_tc() else "fp32")
    unet, tn = _nets()
    rng = np.random.default_rng(2)
    frames = [(_u8(rng, (60, 100, 3)), _u8(rng, (15, 25, 3))) for _ in range(3)]
    st = S2.Stage2(unet, tn, DEV)
    first = [{k: v.copy() for k, v in st.frame(c, a).items()} for c, a in frames]
    st.reset()
    r0 = st.frame(*frames[0])
    r1 = st.frame(torch.from_numpy(frames[1][0]).to(DEV), torch.from_numpy(frames[1][1]))      # device / host tensors
    for k in r0:                                   # r0 is still valid after one more call
        assert r0[k].shape == first[0][k].shape and np.array_equal(r0[k], first[0][k]), k
        assert np.array_equal(r1[k], first[1][k]), k
    assert np.array_equal(st.frame(*frames[2])["final"], first[2]["final"])
    assert not np.array_equal(first[1]["final"], first[1]["filter"])


def test_sixteen_bit_frames_take_the_host_path(tmp_path):
    K.set_conv_precision("tc" if N.lib().b200_device_supports_tc() else "fp32")
    script = _script()
    unet, tn = _nets()
    cn, an = _sequence(str(tmp_path / "in"), 3, (67, 101), (23, 37), dtype=np.uint16)
    assert np.array(Image.open(cn[0])).dtype == np.uint16
    with torch.no_grad():
        host = _dirs(tmp_path / "host")
        _host_loop(unet, tn, cn, an, host)
        d = _dirs(tmp_path / "dev")
        script.run_frames(S2.Stage2(unet, tn, DEV), cn, an, d)
    assert _files(d, 3) == _files(host, 3)
