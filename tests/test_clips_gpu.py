"""A video longer than maximum_number_of_frames fitted as clips (`--clips`, GPU).  A seeded synthetic video of
T = 2M + 1 = 13 frames (M = 6) gives clips of 5, 4 and 4 frames.  Each clip's files match those of a stand-alone run
on a folder holding only its frames (and flows, and mattes): in one process, under torch.distributed.run, and for
the clips of ranks 0..N-1 fitted one after the other in this process.  The loader of a clip equals the loader of such
a folder bit for bit, without reading the flows across clip boundaries; a three-clip run needs no more device memory
than its largest clip; `test.py --clips` runs the whole pipeline.

Two runs of the same script on the same input are not bit-identical: the weight-gradient GEMMs split over CTAs sum
with fp32 atomics and the flow-match rows are compacted in claim order, so the summation order changes from run to
run, and early in a fit the atlas's 2^9 pi encoding turns those last-bit differences into visibly different
renders.  So runs are compared by their atlases (every checkpoint tensor within bounds far below what a different
seed or frame range gives: a different initialisation moves every tensor by about its own norm), and each run's
output frames, alpha mattes and PSNR marker must equal, bit for bit, the in-process evaluation of its own checkpoint
at its own frame numbers.  File names, frame numbers, configs and video frame counts are compared exactly."""
import glob
import json
import os
import shutil
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "all-in-one-deflicker_b200")
if PKG not in sys.path:
    sys.path.insert(0, PKG)

from b200 import _native as N  # noqa: E402
from b200 import atlas as A    # noqa: E402

DEV = torch.device("cuda:0")
M, T, H, W = 6, 13, 96, 128
VID = "long"
CLIPS = [(0, 5), (5, 9), (9, 13)]
# the initial seed of every script process below (torch seeds each process's CPU generator differently otherwise)
SEED = 20261018
WRAPPER = None
# short fits (both regimes of the global rigidity term): run-to-run differences are amplified with every iteration,
# and few iterations keep them far below what a wrong seed or frame range gives
IT = 20
SMALL = dict(maximum_number_of_frames=M, iters_num=IT + 1, evaluate_every=IT, pretrain_iter_number=2, samples_batch=2000,
             stop_global_rigidity=10)


@pytest.fixture(scope="module", autouse=True)
def _seeded_wrapper(tmp_path_factory):
    """`python WRAPPER SEED script args...` runs the script as __main__ with the CPU generator seeded with SEED."""
    global WRAPPER
    WRAPPER = str(tmp_path_factory.mktemp("seeded") / "seeded.py")
    with open(WRAPPER, "w") as f:
        f.write("import runpy, sys\nimport torch\ntorch.manual_seed(int(sys.argv[1]))\nsys.argv = sys.argv[2:]\n"
                "runpy.run_path(sys.argv[0], run_name='__main__')\n")


def _env():
    env = dict(os.environ, PYTHONPATH=PKG, B200_ALLOW_RANDOM_RAFT="1")
    for k in ("WORLD_SIZE", "RANK", "LOCAL_RANK"):
        env.pop(k, None)
    return env


def _torchrun(script, args, cwd, nproc=1, timeout=900):
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--standalone", "--nproc-per-node", str(nproc),
                        WRAPPER, str(SEED), os.path.join(PKG, "src", script)] + args, cwd=str(cwd), env=_env(),
                       capture_output=True, text=True, timeout=timeout)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    return r


def _script(script, args, cwd, timeout=900):
    r = subprocess.run([sys.executable, WRAPPER, str(SEED), os.path.join(PKG, "src", script)] + args, cwd=str(cwd),
                       env=_env(), capture_output=True, text=True, timeout=timeout)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    return r


def _config(work, **kw):
    cfg = json.load(open(os.path.join(PKG, "src", "config", "config_flow_100.json")))
    cfg.update(kw)
    path = str(work / "cfg.json")
    json.dump(cfg, open(path, "w"))
    return cfg, path


def _write_video(folder, n=T):
    """A blurred-noise texture panned 2 px / frame to the left and 1 px / frame up, with a brightness flicker, its
    exact flows (where the pre-pass would write RAFT's: it skips existing pairs) and a moving round matte."""
    import cv2
    folder = str(folder)
    os.makedirs(folder)
    rng = np.random.RandomState(0)
    base = cv2.GaussianBlur(rng.rand(H + 2 * n + 16, W + 4 * n + 16, 3).astype(np.float32), (0, 0), 3.0)
    base = (base - base.min()) / (base.max() - base.min())
    seg, flow = folder + "_seg", folder + "_flow"
    os.makedirs(seg)
    os.makedirs(flow)
    yy, xx = np.mgrid[0:H, 0:W]
    for t in range(n):
        crop = base[8 + t:8 + t + H, 4 + 2 * t:4 + 2 * t + W]
        flick = 1.0 + 0.15 * np.sin(1.7 * t)
        cv2.imwrite(os.path.join(folder, "%05d.png" % t), np.clip(crop * flick * 255.0, 0, 255).astype(np.uint8))
        m = (np.hypot(yy - (H * 0.5 - t), xx - (W * 0.5 - 2 * t)) < H * 0.3).astype(np.uint8) * 255
        cv2.imwrite(os.path.join(seg, "%05d.png" % t), m)
    f12 = np.tile(np.array([-2.0, -1.0], np.float32), (H, W, 1))
    for t in range(n - 1):
        a, b = "%05d.png" % t, "%05d.png" % (t + 1)
        np.save(os.path.join(flow, f"{a}_{b}.npy"), f12)
        np.save(os.path.join(flow, f"{b}_{a}.npy"), -f12)


def _clip_folder(src, dst, clip):
    """Copies of frames [c0, c1) of the video folder `src`, their mattes and the flows of the pairs inside the clip."""
    c0, c1 = clip
    names = ["%05d.png" % t for t in range(c0, c1)]
    for sub in ("", "_seg"):
        os.makedirs(str(dst) + sub)
        for n in names:
            shutil.copy(os.path.join(str(src) + sub, n), os.path.join(str(dst) + sub, n))
    os.makedirs(str(dst) + "_flow")
    for a, b in zip(names[:-1], names[1:]):
        for f in (f"{a}_{b}.npy", f"{b}_{a}.npy"):
            shutil.copy(os.path.join(str(src) + "_flow", f), os.path.join(str(dst) + "_flow", f))


def _marker(folder):
    m = glob.glob(os.path.join(str(folder), "PSNR_*"))
    assert len(m) == 1, m
    return os.path.basename(m[0])


# bounds on the run-to-run differences of a checkpoint: relative Frobenius norm of each parameter tensor / Adam moment
PARAM_REL, MOMENT_REL = 2e-2, 0.3
WORST = {}


def _close_tree(a, b, path="", moments=False):
    """Nested dicts / lists / tensors: same structure, integers and scalars equal, float tensors within PARAM_REL
    (MOMENT_REL under the optimiser's `state`)."""
    assert type(a) is type(b), (path, type(a), type(b))
    if isinstance(a, dict):
        assert set(a) == set(b), path
        for k in a:
            _close_tree(a[k], b[k], f"{path}/{k}", moments or k == "state")
    elif isinstance(a, (list, tuple)):
        assert len(a) == len(b), path
        for i, (x, y) in enumerate(zip(a, b)):
            _close_tree(x, y, f"{path}/{i}", moments)
    elif isinstance(a, torch.Tensor) and a.dim() > 0 and a.is_floating_point():
        assert a.dtype == b.dtype and a.shape == b.shape, path
        r = float((a.double() - b.double()).norm() / max(float(b.double().norm()), 1e-30))
        kind = "moment" if moments else "param"
        WORST[kind] = max(WORST.get(kind, 0.0), r)
        assert r <= (MOMENT_REL if moments else PARAM_REL), (path, r)
    elif isinstance(a, torch.Tensor):
        assert torch.equal(a, b), (path, a, b)
    else:
        assert a == b, (path, a, b)


def _close_checkpoint(a, b):
    _close_tree(torch.load(str(a), weights_only=False), torch.load(str(b), weights_only=False))
    print("clips: largest relative difference of two runs' checkpoint tensors so far", WORST)


def _same_bytes(a, b):
    assert open(str(a), "rb").read() == open(str(b), "rb").read(), (a, b)


def _video_lengths(path):
    import cv2
    cap = cv2.VideoCapture(str(path))
    n = int(cap.get(cv2.CAP_PROP_FRAME_COUNT)) if cap.isOpened() else -1
    cap.release()
    return n


def _files(folder, skip_output=True):
    """Files under `folder` (relative names), with the tensorboard log's host- and time-stamped name and the PSNR
    marker's value left out of the name."""
    out = []
    for p in glob.glob(str(folder / "**" / "*"), recursive=True):
        rel = os.path.relpath(p, str(folder))
        if os.path.isdir(p) or (skip_output and rel.startswith("output" + os.sep)):
            continue
        for stamped in ("events.out.tfevents", "PSNR_"):
            if os.path.basename(rel).startswith(stamped):
                rel = os.path.join(os.path.dirname(rel), stamped)
        out.append(rel)
    return sorted(out)


def _check_clip(res, clip, ref, data, cfg, tmp, seg=False):
    """Clip `clip` of a --clips run whose stage_1 folder is `res`, against `ref`, the stage_1 folder of a run that
    fitted the same atlas (stand-alone on the clip's folder, or the clip's folder of another --clips run): the same
    files, config and video lengths, checkpoints within bounds, and frames, mattes and PSNR marker equal to the
    evaluation of its own checkpoint, written at the clip's frame numbers."""
    from src.models.stage_1 import evaluate as E
    c0, c1 = clip
    n, d, it = c1 - c0, res / A.clip_name(clip), "%06d" % IT
    assert not os.path.exists(str(d / "output"))
    assert _files(d) == _files(ref) and len(_files(d)) >= (8 if seg else 10), (_files(d), _files(ref))
    _same_bytes(d / "config.json", ref / "config.json")
    for v in glob.glob(str(ref / "**" / "*.mp4"), recursive=True):
        assert _video_lengths(d / os.path.relpath(v, str(ref))) == _video_lengths(v), v
    _close_checkpoint(d / "checkpoint", ref / "checkpoint")
    if seg:
        _close_checkpoint(d / it / "checkpoint", ref / it / "checkpoint")
    ck = torch.load(str(d / "checkpoint"), weights_only=False)
    video, frames = A.DeviceVideo.from_files(data, data.parent, VID, H, W, M, DEV, clip=clip)
    precision = N.PREC_TC if N.lib().b200_device_supports_tc() else N.PREC_FP32
    out = tmp / f"eval_{c0}"
    if seg:
        from b200 import seg as SG
        tr = SG.SegTrainer(video, None, cfg, precision=precision, device=DEV, resx=W)
        tr.load_state(dict(atlas=ck["F_atlas_state_dict"], mapping1=ck["model_F_mapping1_state_dict"],
                           mapping2=ck["model_F_mapping2_state_dict"], alpha=ck["model_F_alpha_state_dict"]))
        psnr = E.evaluate_model(tr, W, H, n, frames, str(out), IT, save_checkpoint=False,
                                output_folder=str(out / "frames"), frame_offset=c0)
        for f in range(n):
            _same_bytes(d / it / "alpha" / ("%05d.png" % f), out / it / "alpha" / ("%05d.png" % f))
    else:
        tr = A.AtlasTrainer(video, cfg, precision=precision, device=DEV, resx=W)
        tr.load_state(ck["model_F_mapping1_state_dict"], ck["F_atlas_state_dict"])
        psnr = E.evaluate_model_single(tr, W, H, n, frames, str(out), IT, VID, save_checkpoint=False,
                                       output_folder=str(out / "frames"), frame_offset=c0)
    tr.release()
    assert sorted(os.listdir(str(out / "frames"))) == ["%05d.png" % t for t in range(c0, c1)]
    for t in range(c0, c1):
        _same_bytes(res / "output" / ("%05d.png" % t), out / "frames" / ("%05d.png" % t))
    assert _marker(d / it) == "PSNR_%f" % psnr


def _check_clip_runs(res, refs, data, cfg, tmp, seg=False):
    assert sorted(os.listdir(str(res / "output"))) == ["%05d.png" % t for t in range(T)]
    assert sorted(p for p in os.listdir(str(res)) if p != "output") == [A.clip_name(c) for c in CLIPS]
    for clip, ref in zip(CLIPS, refs):
        _check_clip(res, clip, ref, data, cfg, tmp, seg)


@pytest.fixture(scope="module")
def clip_runs(tmp_path_factory):
    """The atlas script with --clips on the 13-frame video, and stand-alone on each clip's folder."""
    work = tmp_path_factory.mktemp("clips_atlas")
    _write_video(work / "data" / "test" / VID)
    cfg, path = _config(work, **SMALL)
    _script("stage1_neural_atlas.py", ["--vid_name", VID, "--root", "data/test/", "--down", "1", "--config", path,
                                       "--clips"], work)
    alone = []
    for k, clip in enumerate(CLIPS):
        w = tmp_path_factory.mktemp(f"clip_alone{k}")
        _clip_folder(work / "data" / "test" / VID, w / "data" / "test" / VID, clip)
        _script("stage1_neural_atlas.py", ["--vid_name", VID, "--root", "data/test/", "--down", "1", "--config", path], w)
        alone.append(w / "results" / VID / "stage_1")
    return work, cfg, path, alone


def test_loader_of_a_clip_equals_a_folder_of_the_clip(tmp_path):
    src = tmp_path / "video" / VID
    _write_video(src)
    for clip in (CLIPS[0], CLIPS[1], CLIPS[2]):
        _clip_folder(src, tmp_path / f"alone{clip[0]}" / VID, clip)
    for c0, c1 in CLIPS[1:]:               # the flows across the clip boundaries are never read
        for f in ("%05d.png_%05d.png.npy" % (c0 - 1, c0), "%05d.png_%05d.png.npy" % (c0, c0 - 1)):
            os.remove(os.path.join(str(src) + "_flow", f))
    for clip in CLIPS:
        one = tmp_path / f"alone{clip[0]}" / VID
        got, got_frames = A.DeviceVideo.from_files(src, src.parent, VID, H, W, M, DEV, clip=clip)
        want, want_frames = A.DeviceVideo.from_files(one, one.parent, VID, H, W, M, DEV)
        assert (got.T, got.t_begin, got.t_end) == (want.T, want.t_begin, want.t_end) == (clip[1] - clip[0], 0,
                                                                                        clip[1] - clip[0])
        for a, b in ((got.records, want.records), (got.bits_f, want.bits_f), (got.bits_b, want.bits_b),
                     (got_frames, want_frames)):
            assert a.shape == b.shape and torch.equal(a, b)
        assert int(got.bits_f.ne(0).sum()) > 0
    with pytest.raises(N.B200Error, match="outside"):
        A.DeviceVideo.from_files(src, src.parent, VID, H, W, M, DEV, clip=(9, 14))


def test_atlas_script_clips_equal_stand_alone_runs(clip_runs, tmp_path):
    work, cfg, path, alone = clip_runs
    res = work / "results" / VID / "stage_1"
    _check_clip_runs(res, alone, work / "data" / "test" / VID, cfg, tmp_path)
    # artefact names keep the video's name
    assert os.path.exists(str(res / A.clip_name(CLIPS[0]) / ("%06d" % IT) / f"reconstruction_{VID}.mp4"))


def test_atlas_script_clips_under_torchrun_equal_one_process(clip_runs, tmp_path):
    work, cfg, path, _ = clip_runs
    data = tmp_path / "data" / "test" / VID
    _write_video(data)
    _torchrun("stage1_neural_atlas.py", ["--vid_name", VID, "--root", "data/test/", "--down", "1", "--config", path,
                                         "--clips"], tmp_path)
    one = work / "results" / VID / "stage_1"
    _check_clip_runs(tmp_path / "results" / VID / "stage_1", [one / A.clip_name(c) for c in CLIPS], data, cfg, tmp_path)


def _args(vid_path, no_artefacts=False):
    return types.SimpleNamespace(vid_path=str(vid_path), down=1, no_artefacts=no_artefacts)


def test_rank_clip_lists_in_one_process_equal_one_rank(clip_runs, tmp_path, monkeypatch):
    """Ranks 0..N-1 of N = 2 and 3 fit their clips one after the other on this GPU; together they write what the
    one-process run wrote."""
    from src.models.stage_1 import driver as D
    from src.stage1_neural_atlas import VARIANT
    work, cfg, _, _ = clip_runs
    one = work / "results" / VID / "stage_1"
    for world in (2, 3):
        w = tmp_path / f"world{world}"
        data = w / "data" / "test" / VID
        _write_video(data)
        monkeypatch.chdir(w)
        for rank in range(world):
            D.fit_clips(VARIANT, cfg, _args(data), A.rank_clips(CLIPS, rank, world), DEV, SEED)
        _check_clip_runs(w / "results" / VID / "stage_1", [one / A.clip_name(c) for c in CLIPS], data, cfg, w)


def test_clip_run_peak_memory_is_the_largest_clips(clip_runs, tmp_path, monkeypatch):
    """max_memory_allocated of the three-clip run against a stand-alone fit of its largest clip (5 frames), in this
    process; the library's cached tensor-core job tables of every clip are released with its trainer."""
    from src.models.stage_1 import driver as D
    from src.stage1_neural_atlas import VARIANT
    work, cfg, _, _ = clip_runs
    w = tmp_path / "mem"
    _write_video(w / "data" / "test" / VID)
    _clip_folder(w / "data" / "test" / VID, tmp_path / "mem_one" / "data" / "test" / VID, CLIPS[0])
    monkeypatch.chdir(tmp_path / "mem_one")
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    tables = N.lib().b200_tc_cached_tables()
    torch.cuda.reset_peak_memory_stats(DEV)
    torch.manual_seed(SEED)
    D.fit(VARIANT, cfg, _args(tmp_path / "mem_one" / "data" / "test" / VID, True), DEV)
    largest = torch.cuda.max_memory_allocated(DEV)
    assert N.lib().b200_tc_cached_tables() == tables
    monkeypatch.chdir(w)
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats(DEV)
    D.fit_clips(VARIANT, cfg, _args(w / "data" / "test" / VID, True), CLIPS, DEV, SEED)
    three = torch.cuda.max_memory_allocated(DEV)
    print(f"peak device memory: three clips {three} B, largest clip alone {largest} B")
    assert three <= 1.03 * largest, (three, largest)
    assert N.lib().b200_tc_cached_tables() == tables
    assert len(os.listdir(str(w / "results" / VID / "stage_1" / "output"))) == T


def test_seg_script_clips_equal_stand_alone_runs(tmp_path):
    work = tmp_path / "clips"
    _write_video(work / "data" / "test" / VID)
    cfg, path = _config(tmp_path, **dict(SMALL, samples_batch=1500))
    args = ["--vid_name", VID, "--root", "data/test/", "--down", "1", "--class_name", "person", "--config", path]
    _script("stage1_neural_atlas_seg.py", args + ["--clips"], work)
    alone = []
    for k, clip in enumerate(CLIPS):
        w = tmp_path / f"alone{k}"
        _clip_folder(work / "data" / "test" / VID, w / "data" / "test" / VID, clip)
        _script("stage1_neural_atlas_seg.py", args, w)
        alone.append(w / "results" / VID / "stage_1")
    _check_clip_runs(work / "results" / VID / "stage_1", alone, work / "data" / "test" / VID, cfg, tmp_path, seg=True)
    # a matte folder short of the last clip's frames is refused, naming the clip, before any clip is fitted
    shutil.rmtree(str(work / "results"))
    os.remove(str(work / "data" / "test" / (VID + "_seg") / "00012.png"))
    r = subprocess.run([sys.executable, os.path.join(PKG, "src", "stage1_neural_atlas_seg.py")] + args + ["--clips"],
                       cwd=str(work), env=_env(), capture_output=True, text=True, timeout=600)
    assert r.returncode != 0 and "clip_00009_00013" in r.stderr
    assert not os.path.exists(str(work / "results" / VID / "stage_1" / "output"))


def test_driver_with_clips_end_to_end(tmp_path):
    from src.models.network_filter import UNet
    from src.models.network_local import TransformNet
    _write_video(tmp_path / "data" / "test" / VID)
    cfg, path = _config(tmp_path, **SMALL)
    # test.py starts stage 1 with the shipped config name: give it this one under that name in a copy of the package
    pkg = tmp_path / "pkg"
    shutil.copytree(PKG, str(pkg), ignore=shutil.ignore_patterns("__pycache__"))
    shutil.copy(path, str(pkg / "src" / "config" / "config_flow_100.json"))
    os.makedirs(str(tmp_path / "pretrained_weights"))
    torch.manual_seed(0)
    torch.save(UNet(in_channels=6, out_channels=3, init_features=32).state_dict(),
               str(tmp_path / "pretrained_weights" / "neural_filter.pth"))
    tn = TransformNet(types.SimpleNamespace(nf=32, norm="IN", model="TransformNet", blocks=5), nc_in=12, nc_out=3)
    torch.save(tn.state_dict(), str(tmp_path / "pretrained_weights" / "local_refinement_net.pth"))
    env = dict(_env(), PYTHONPATH=str(pkg))
    r = subprocess.run([sys.executable, str(pkg / "test.py"), "--video_frame_folder", VID, "--clips"], cwd=str(tmp_path),
                       env=env, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    res = tmp_path / "results" / VID
    assert sorted(p for p in os.listdir(str(res / "stage_1")) if p.startswith("clip_")) == [A.clip_name(c) for c in CLIPS]
    for sub in ("stage_1/output", "neural_filter/concat", "neural_filter/output", "final/output"):
        assert len(glob.glob(str(res / sub / "*.png"))) == T, sub
