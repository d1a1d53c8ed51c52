"""The stage-1 scripts under a process group (GPU): both variants started by torch.distributed.run meet the on-disk
contract of the single-GPU scripts and write what an in-process whole-video evaluation of their checkpoint writes; a
2- and 3-way frame-sharded evaluation emulated in one process equals the whole-video one; `test.py --gpus 2` end to
end on a node with two GPUs."""
import glob
import json
import os
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

from test_pipeline_gpu import _write_video

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "all-in-one-deflicker_b200")
if PKG not in sys.path:
    sys.path.insert(0, PKG)

from b200 import _native as N  # noqa: E402
from b200 import atlas as A    # noqa: E402
from b200 import seg as SG     # noqa: E402
from src.models.stage_1 import evaluate as E  # noqa: E402

DEV = torch.device("cuda:0")


def _torchrun(script, args, cwd, nproc=1, timeout=900):
    env = dict(os.environ, PYTHONPATH=PKG, B200_ALLOW_RANDOM_RAFT="1")
    for k in ("WORLD_SIZE", "RANK", "LOCAL_RANK"):
        env.pop(k, None)
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--standalone", "--nproc-per-node", str(nproc),
                        os.path.join(PKG, "src", script)] + args, cwd=str(cwd), env=env, capture_output=True, text=True,
                       timeout=timeout)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    return r


def _config(work, **kw):
    cfg = json.load(open(os.path.join(PKG, "src", "config", "config_flow_100.json")))
    cfg.update(kw)
    path = str(work / "cfg.json")
    json.dump(cfg, open(path, "w"))
    return cfg, path


def _precision():
    return N.PREC_TC if N.lib().b200_device_supports_tc() else N.PREC_FP32


def _marker(folder):
    m = glob.glob(os.path.join(str(folder), "PSNR_*"))
    assert len(m) == 1, m
    return os.path.basename(m[0])


def _same_pngs(dir_a, dir_b, n):
    a, b = sorted(glob.glob(os.path.join(str(dir_a), "*.png"))), sorted(glob.glob(os.path.join(str(dir_b), "*.png")))
    assert len(a) == len(b) == n
    for x, y in zip(a, b):
        assert os.path.basename(x) == os.path.basename(y)
        assert open(x, "rb").read() == open(y, "rb").read(), x


def _atlas_trainer(work, vid, cfg, ck, t_begin=0, t_end=None):
    data = work / "data" / "test" / vid
    video, frames = A.DeviceVideo.from_files(data, data.parent, vid, 128, 192, cfg["maximum_number_of_frames"], DEV,
                                             t_begin=t_begin, t_end=t_end, decode_all=t_end is None)
    tr = A.AtlasTrainer(video, cfg, precision=_precision(), device=DEV, resx=192)
    tr.load_state(ck["model_F_mapping1_state_dict"], ck["F_atlas_state_dict"])
    return tr, frames


@pytest.fixture(scope="module")
def atlas_run(tmp_path_factory):
    """The atlas script on one rank of torch.distributed.run, on the tiny clip of test_pipeline_gpu."""
    work = tmp_path_factory.mktemp("mg_atlas")
    vid = "tiny"
    _write_video(str(work / "data" / "test" / vid))
    cfg, path = _config(work, iters_num=201, evaluate_every=200, pretrain_iter_number=2, samples_batch=2000,
                        stop_global_rigidity=100)
    _torchrun("stage1_neural_atlas.py", ["--vid_name", vid, "--root", "data/test/", "--down", "1", "--config", path], work)
    return work, vid, cfg


def test_atlas_script_under_torchrun_meets_the_contract(atlas_run, tmp_path):
    import cv2
    work, vid, cfg = atlas_run
    assert len(glob.glob(str(work / "data" / "test" / (vid + "_flow") / "*.npy"))) == 10
    res = work / "results" / vid / "stage_1"
    ck = torch.load(str(res / "checkpoint"), weights_only=False)
    assert set(ck) == {"F_atlas_state_dict", "iteration", "model_F_mapping1_state_dict", "optimizer_all_state_dict"}
    assert ck["iteration"] == 200 and len(ck["F_atlas_state_dict"]) == 16 and len(ck["model_F_mapping1_state_dict"]) == 12
    assert len(ck["optimizer_all_state_dict"]["param_groups"]) == 2
    for name, n in (("000200/reconstruction_tiny.mp4", 6), ("000200/residuals_tiny.mp4", 6),
                    ("000200/uv_1_tiny.mp4", 6), ("000200/global_info_tiny.mp4", 6), ("input_video.mp4", 6)):
        cap = cv2.VideoCapture(str(res / name))
        assert cap.isOpened() and int(cap.get(cv2.CAP_PROP_FRAME_COUNT)) == n, name
        cap.release()
    assert glob.glob(str(res / "events.out.tfevents.*"))
    # the frames and PSNR of an in-process whole-video evaluation of the written checkpoint
    tr, frames = _atlas_trainer(work, vid, cfg, ck)
    ref = tmp_path / "ref"
    psnr = E.evaluate_model_single(tr, 192, 128, 6, frames, str(ref), 200, vid, save_checkpoint=False)
    _same_pngs(res / "output", ref / "output", 6)
    assert _marker(res / "000200") == "PSNR_%f" % psnr


def test_sharded_evaluation_equals_whole_video(atlas_run, tmp_path):
    """2- and 3-way frame blocks evaluated one after the other in this process, merged as rank 0 merges them."""
    work, vid, cfg = atlas_run
    ck = torch.load(str(work / "results" / vid / "stage_1" / "checkpoint"), weights_only=False)
    tr, frames = _atlas_trainer(work, vid, cfg, ck)
    whole = tmp_path / "whole"
    psnr = E.evaluate_model_single(tr, 192, 128, 6, frames, str(whole), 200, vid, save_checkpoint=False)
    want_images = []
    for f in range(6):
        img = tr.render_frame(f, 128, 192, 6).cpu().numpy()
        uv, rig, flow = tr.eval_maps(f)
        want_images.append(E.artefact_images(frames[:, :, :, f].numpy(), img, uv.cpu().numpy(), rig.cpu().numpy(),
                                             flow.cpu().numpy()))
    for world in (2, 3):
        out = tmp_path / f"shard{world}"
        os.makedirs(str(out / "output"))
        os.makedirs(str(out / "000200"))
        psnrs, payloads = [], []
        for r in range(world):
            t0, t1 = A.frame_range(r, world, 6)
            shard, none = _atlas_trainer(work, vid, cfg, ck, t0, t1)
            assert none is None
            p, pl = E.evaluate_block_single(shard, 192, 128, 6, str(out), artefacts=True)
            psnrs += p
            payloads += pl
        assert len(psnrs) == len(payloads) == 6
        _same_pngs(out / "output", whole / "output", 6)
        assert abs(float(np.mean(psnrs)) - psnr) < 1e-9
        for f in range(6):
            got = E._unpack(payloads[f], 192, 128)
            for g, w in zip(got, want_images[f]):
                assert np.array_equal(g, w), f
        mean = E.write_evaluation_single(tr, 192, 128, 6, str(out), 200, psnrs, vid, payloads)
        assert abs(mean - psnr) < 1e-9 and _marker(out / "000200") == "PSNR_%f" % psnr
        assert len(glob.glob(str(out / "000200" / "*.mp4"))) == 4


def test_seg_script_under_torchrun_meets_the_contract(tmp_path):
    import cv2
    work = tmp_path
    vid = "tinyseg"
    T, H, W = 5, 96, 128
    _write_video(str(work / "data" / "test" / vid), T=T, H=H, W=W)
    seg_dir = str(work / "data" / "test" / (vid + "_seg"))
    os.makedirs(seg_dir)
    yy, xx = np.mgrid[0:H, 0:W]
    for t in range(T):
        m = (np.hypot(yy - (H * 0.5 - t), xx - (W * 0.5 - 2 * t)) < H * 0.3).astype(np.uint8) * 255
        cv2.imwrite(os.path.join(seg_dir, "%05d.png" % t), m)
    cfg, path = _config(work, iters_num=101, evaluate_every=100, pretrain_iter_number=2, samples_batch=1500,
                        stop_global_rigidity=50)
    _torchrun("stage1_neural_atlas_seg.py", ["--vid_name", vid, "--root", "data/test/", "--down", "1", "--class_name",
                                             "person", "--config", path], work)
    assert len(glob.glob(str(work / "data" / "test" / (vid + "_flow") / "*.npy"))) == 2 * (T - 1)
    res = work / "results" / vid / "stage_1"
    ck = torch.load(str(res / "checkpoint"), weights_only=False)
    assert set(ck) == {"F_atlas_state_dict", "iteration", "model_F_mapping1_state_dict", "model_F_mapping2_state_dict",
                       "model_F_alpha_state_dict", "optimizer_all_state_dict"}
    assert ck["iteration"] == 100 and len(ck["optimizer_all_state_dict"]["param_groups"]) == 4
    assert os.path.exists(str(res / "000100" / "checkpoint"))
    data = work / "data" / "test" / vid
    video, frames = A.DeviceVideo.from_files(data, data.parent, vid, H, W, cfg["maximum_number_of_frames"], DEV)
    tr = SG.SegTrainer(video, None, cfg, precision=_precision(), device=DEV, resx=W)
    tr.load_state(dict(atlas=ck["F_atlas_state_dict"], mapping1=ck["model_F_mapping1_state_dict"],
                       mapping2=ck["model_F_mapping2_state_dict"], alpha=ck["model_F_alpha_state_dict"]))
    ref = tmp_path / "ref"
    psnr = E.evaluate_model(tr, W, H, T, frames, str(ref), 100, save_checkpoint=False)
    _same_pngs(res / "output", ref / "output", T)
    _same_pngs(res / "000100" / "alpha", ref / "000100" / "alpha", T)
    assert _marker(res / "000100") == "PSNR_%f" % psnr
    # the device PSNR of the sharded evaluation agrees with the host one to 1e-9
    blk = tmp_path / "blk"
    os.makedirs(str(blk / "output"))
    os.makedirs(str(blk / "000100" / "alpha"))
    assert abs(float(np.mean(E.evaluate_block_seg(tr, W, H, T, str(blk), 100))) - psnr) < 1e-9


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="test.py --gpus 2 needs two GPUs on the node")
def test_driver_on_two_gpus_end_to_end(tmp_path):
    from src.models.network_filter import UNet
    from src.models.network_local import TransformNet
    env = dict(os.environ, PYTHONPATH=PKG, B200_ALLOW_RANDOM_RAFT="1")
    for k in ("WORLD_SIZE", "RANK", "LOCAL_RANK"):
        env.pop(k, None)
    # flows of a one-GPU pre-pass of the same clip (same kernels, same inputs, same random-init RAFT)
    one = tmp_path / "one" / "clip"
    _write_video(str(one))
    r = subprocess.run([sys.executable, os.path.join(PKG, "src", "preprocess_optical_flow.py"), "--vid-path", str(one)],
                       cwd=str(tmp_path), env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    _write_video(str(tmp_path / "clip"))
    os.makedirs(str(tmp_path / "pretrained_weights"))
    torch.manual_seed(0)
    torch.save(UNet(in_channels=6, out_channels=3, init_features=32).state_dict(),
               str(tmp_path / "pretrained_weights" / "neural_filter.pth"))
    tn = TransformNet(types.SimpleNamespace(nf=32, norm="IN", model="TransformNet", blocks=5), nc_in=12, nc_out=3)
    torch.save(tn.state_dict(), str(tmp_path / "pretrained_weights" / "local_refinement_net.pth"))
    r = subprocess.run([sys.executable, os.path.join(PKG, "test.py"), "--video_frame_folder", "clip", "--gpus", "2"],
                       cwd=str(tmp_path), env=env, capture_output=True, text=True, timeout=3000)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    got = sorted(glob.glob(str(tmp_path / "data" / "test" / "clip_flow" / "*.npy")))
    want = sorted(glob.glob(str(tmp_path / "one" / "clip_flow" / "*.npy")))
    assert [os.path.basename(p) for p in got] == [os.path.basename(p) for p in want] and len(got) == 10
    for a, b in zip(got, want):
        assert open(a, "rb").read() == open(b, "rb").read(), a
    res = tmp_path / "results" / "clip"
    assert len(glob.glob(str(res / "stage_1" / "output" / "*.png"))) == 6
    assert len(glob.glob(str(res / "final" / "output" / "*.png"))) == 6
