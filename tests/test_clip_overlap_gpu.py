"""Overlapping clips on the GPU (`--clips --clip_overlap V`).

b200_blend_frames against a float64 numpy restatement, bit for bit in fp32 and in 8 bits, at 1, 255 and 1080p x 3
values, at w = 0 and 1 (a and b exactly) and inside, on values that land exactly on 8-bit steps and as a graph replay;
and its argument checks.

Both stage-1 scripts with --clips --clip_overlap 2 on a seeded 15-frame video with M = 7: clips [0, 7), [5, 11) and
[9, 15), seams [5, 7) and [9, 11).  Each clip matches a stand-alone run on a folder holding only its frames (files,
config, checkpoint within the bounds of tests/test_clips_gpu.py, PSNR marker and mattes of its own checkpoint's
evaluation); every frame a clip renders alone equals its evaluation bit for bit, and every shared frame equals the
restated blend of the two checkpoints' renders at w = 1/3 and 2/3.  Under torch.distributed.run and for two ranks
emulated in one process the stitch writes the same frames from the same checkpoints; a run with no evaluation writes
no frame; `test.py --clips --clip_overlap 2 --evaluate_flicker` runs end to end."""
import glob
import json
import os
import shutil
import subprocess
import sys
import types

import cv2
import numpy as np
import pytest
import torch

import test_clips_gpu as CG

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "all-in-one-deflicker_b200")
if PKG not in sys.path:
    sys.path.insert(0, PKG)

from b200 import _native as N  # noqa: E402
from b200 import atlas as A    # noqa: E402

DEV = torch.device("cuda:0")
M, V, T, H, W = 7, 2, 15, CG.H, CG.W
VID = CG.VID
PLAN = [(0, 7), (5, 11), (9, 15)]
SEAMS = [(5, 7), (9, 11)]
IT = CG.IT
SMALL = dict(CG.SMALL, maximum_number_of_frames=M)
SEED = CG.SEED
WRAPPER = None


@pytest.fixture(scope="module", autouse=True)
def _seeded_wrapper(tmp_path_factory):
    """`python WRAPPER SEED script args...` runs the script as __main__ with the CPU generator seeded with SEED."""
    global WRAPPER
    WRAPPER = str(tmp_path_factory.mktemp("seeded") / "seeded.py")
    with open(WRAPPER, "w") as f:
        f.write("import runpy, sys\nimport torch\ntorch.manual_seed(int(sys.argv[1]))\nsys.argv = sys.argv[2:]\n"
                "runpy.run_path(sys.argv[0], run_name='__main__')\n")


def _run(cmd, cwd, timeout=900):
    r = subprocess.run(cmd, cwd=str(cwd), env=CG._env(), capture_output=True, text=True, timeout=timeout)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    return r


def _script(script, args, cwd):
    return _run([sys.executable, WRAPPER, str(SEED), os.path.join(PKG, "src", script)] + args, cwd)


# ---------------------------------------------------------------------------------------------------------------------
# the kernel

def restated(a, b, w):
    """The kernel's arithmetic in numpy: float64 products and sum, one rounding each, fp32 once; then the renders'
    8-bit truncation (int conversion, then the low byte)."""
    a64, b64 = np.asarray(a, np.float32).astype(np.float64), np.asarray(b, np.float32).astype(np.float64)
    o = ((1.0 - w) * a64 + w * b64).astype(np.float32)
    return o, (o.astype(np.float64) * 255.0).astype(np.int64).astype(np.uint8)


def _blend(a, b, w):
    out, u8 = A.blend_frames(a, b, w, want_u8=True)
    torch.cuda.synchronize()
    return out.cpu().numpy(), u8.cpu().numpy()


def _check(a, b, w):
    got_o, got_u = _blend(a, b, w)
    want_o, want_u = restated(a.cpu().numpy(), b.cpu().numpy(), w)
    assert np.array_equal(got_o.view(np.uint32), want_o.view(np.uint32)), w
    assert np.array_equal(got_u, want_u), w
    return got_o, got_u


@pytest.mark.parametrize("n", [1, 3 * 17 * 5, 1080 * 1920 * 3])
@pytest.mark.parametrize("w", [0.0, 1.0, 1 / 3, 2 / 3, 0.5, 1 / 9, 8 / 9, 0.123456789])
def test_blend_equals_the_restatement(n, w):
    g = torch.Generator(device=DEV).manual_seed(n)
    a = torch.rand(n, generator=g, device=DEV)
    b = torch.rand(n, generator=g, device=DEV)
    o, u8 = _check(a, b, w)
    if w == 0.0:
        assert np.array_equal(o.view(np.uint32), a.cpu().numpy().view(np.uint32))
    if w == 1.0:
        assert np.array_equal(o.view(np.uint32), b.cpu().numpy().view(np.uint32))


def test_blend_out_of_range_values_follow_the_restatement():
    """Values outside [0, 1] (not produced by a render, but allowed): the 8-bit value is the low byte of the int."""
    g = torch.Generator(device=DEV).manual_seed(5)
    a = torch.rand(4096, generator=g, device=DEV) * 4 - 2
    b = torch.rand(4096, generator=g, device=DEV) * 4 - 2
    for w in (0.0, 0.25, 1.0):
        _check(a, b, w)


def test_blend_on_exact_8_bit_steps():
    """k / 255 in fp32 and its two neighbours, for every k: where (double)o * 255 lands just below or on k."""
    steps = (np.arange(256, dtype=np.float64) / 255.0).astype(np.float32)
    vals = np.concatenate([steps, np.nextafter(steps, np.float32(-1)), np.nextafter(steps, np.float32(2))])
    a = torch.from_numpy(vals).to(DEV)
    b = torch.from_numpy(vals[::-1].copy()).to(DEV)
    for w in (0.0, 1.0, 1 / 3, 0.5):
        _check(a, b, w)
    _, u8 = _check(a, a, 0.0)
    assert np.array_equal(u8[:256], (steps.astype(np.float64) * 255.0).astype(np.int64).astype(np.uint8))
    # a blend of equal values that land on a step: the truncation is applied to the blended fp32 value
    _check(a, a, 1 / 3)


def test_blend_out_or_u8_alone_and_the_same_bits():
    g = torch.Generator(device=DEV).manual_seed(9)
    a, b = torch.rand(777, generator=g, device=DEV), torch.rand(777, generator=g, device=DEV)
    both_o, both_u = _blend(a, b, 0.3)
    only_o, none_u = A.blend_frames(a, b, 0.3)
    none_o, only_u = A.blend_frames(a, b, 0.3, want_out=False, want_u8=True)
    assert none_u is None and none_o is None
    assert np.array_equal(only_o.cpu().numpy().view(np.uint32), both_o.view(np.uint32))
    assert np.array_equal(only_u.cpu().numpy(), both_u)


def test_blend_as_a_graph_replay():
    n = 1080 * 1920 * 3
    g = torch.Generator(device=DEV).manual_seed(11)
    a, b = torch.empty(n, device=DEV), torch.empty(n, device=DEV)
    out, u8 = torch.empty(n, device=DEV), torch.empty(n, dtype=torch.uint8, device=DEV)
    A.blend_frames(a.fill_(0.5), b.fill_(0.25), 0.4, out, u8, want_u8=True)    # warm-up
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        A.blend_frames(a, b, 0.4, out, u8, want_u8=True)
    for _ in range(3):
        a.copy_(torch.rand(n, generator=g, device=DEV))
        b.copy_(torch.rand(n, generator=g, device=DEV))
        graph.replay()
        torch.cuda.synchronize()
        want_o, want_u = restated(a.cpu().numpy(), b.cpu().numpy(), 0.4)
        assert np.array_equal(out.cpu().numpy().view(np.uint32), want_o.view(np.uint32))
        assert np.array_equal(u8.cpu().numpy(), want_u)


def test_blend_argument_checks():
    lib = N.lib()
    a, b = torch.rand(8, device=DEV), torch.rand(8, device=DEV)
    out, u8 = torch.empty(8, device=DEV), torch.empty(8, dtype=torch.uint8, device=DEV)
    st = N.current_stream()
    cases = [((None, N.ptr(b), 8, 0.5, N.ptr(out), None), "null input"),
             ((N.ptr(a), None, 8, 0.5, N.ptr(out), None), "null input"),
             ((N.ptr(a), N.ptr(b), 8, 0.5, None, None), "both NULL"),
             ((N.ptr(a), N.ptr(b), 0, 0.5, N.ptr(out), None), "n must be >= 1"),
             ((N.ptr(a), N.ptr(b), -3, 0.5, N.ptr(out), None), "n must be >= 1")]
    for w in (-1e-300, 1.0000000000000002, float("nan"), float("inf"), float("-inf")):
        cases.append(((N.ptr(a), N.ptr(b), 8, w, N.ptr(out), N.ptr(u8)), "w must be finite and in [0, 1]"))
    out.fill_(7.0)
    for args, msg in cases:
        assert lib.b200_blend_frames(*args, st) != 0, args
        assert msg in N.last_error(), (args, N.last_error())
    torch.cuda.synchronize()
    assert bool((out == 7.0).all())                 # a refused call launches nothing
    with pytest.raises(N.B200Error, match="both NULL"):
        A.blend_frames(a, b, 0.5, want_out=False)
    with pytest.raises(N.B200Error, match="fp32 device tensors"):
        A.blend_frames(a, b[:4], 0.5)


# ---------------------------------------------------------------------------------------------------------------------
# the scripts

def _render_trainer(ck_path, cfg, seg):
    ck = torch.load(str(ck_path), weights_only=False)
    precision = N.PREC_TC if N.lib().b200_device_supports_tc() else N.PREC_FP32
    if seg:
        from b200 import seg as SG
        tr = SG.SegTrainer(None, None, cfg, precision=precision, device=DEV, resx=W)
        tr.load_state(dict(atlas=ck["F_atlas_state_dict"], mapping1=ck["model_F_mapping1_state_dict"],
                           mapping2=ck["model_F_mapping2_state_dict"], alpha=ck["model_F_alpha_state_dict"]))
    else:
        tr = A.AtlasTrainer(None, cfg, precision=precision, device=DEV, resx=W)
        tr.load_state(ck["model_F_mapping1_state_dict"], ck["F_atlas_state_dict"])
    return tr


def _render(tr, f, n):
    out = tr.render_frame(f, H, W, n)
    return (out[0] if isinstance(out, tuple) else out).cpu().numpy()


def _read_rgb(path):
    return cv2.cvtColor(cv2.imread(str(path), cv2.IMREAD_UNCHANGED), cv2.COLOR_BGR2RGB)


def _check_seams(res, cfg, seg):
    """Every shared frame of `res`/output equals the restated blend of its two clips' checkpoint renders."""
    for k, (a, b) in enumerate(SEAMS):
        (l0, l1), (r0, r1) = PLAN[k], PLAN[k + 1]
        left = _render_trainer(res / A.clip_name(PLAN[k]) / "checkpoint", cfg, seg)
        right = _render_trainer(res / A.clip_name(PLAN[k + 1]) / "checkpoint", cfg, seg)
        for j, w in enumerate(A.seam_weights(b - a)):
            assert w == (j + 1) / 3
            t = a + j
            x, y = _render(left, t - l0, l1 - l0), _render(right, t - r0, r1 - r0)
            _, want = restated(x, y, w)
            got = _read_rgb(res / "output" / ("%05d.png" % t))
            assert np.array_equal(got, want), (k, t)
            # a true cross-fade: neither atlas's frame alone
            assert not np.array_equal(got, restated(x, y, 0.0)[1]) and not np.array_equal(got, restated(x, y, 1.0)[1])
        left.release()
        right.release()


def _check_clip(res, k, ref, data, cfg, tmp, seg):
    """Clip k against the stand-alone run `ref`: files, config, checkpoint within bounds, marker and mattes of its own
    checkpoint's evaluation, and the frames it renders alone bit for bit."""
    from src.models.stage_1 import evaluate as E
    clip = PLAN[k]
    c0, c1 = clip
    n, d, it = c1 - c0, res / A.clip_name(clip), "%06d" % IT
    assert CG._files(d) == CG._files(ref), (CG._files(d), CG._files(ref))
    CG._same_bytes(d / "config.json", ref / "config.json")
    CG._close_checkpoint(d / "checkpoint", ref / "checkpoint")
    _, frames = A.DeviceVideo.from_files(data, data.parent, VID, H, W, M, DEV, clip=clip)
    tr = _render_trainer(d / "checkpoint", cfg, seg)
    out = tmp / f"eval_{c0}"
    if seg:
        CG._close_checkpoint(d / it / "checkpoint", ref / it / "checkpoint")
        psnr = E.evaluate_model(tr, W, H, n, frames, str(out), IT, save_checkpoint=False,
                                output_folder=str(out / "frames"), frame_offset=c0)
        for f in range(n):
            CG._same_bytes(d / it / "alpha" / ("%05d.png" % f), out / it / "alpha" / ("%05d.png" % f))
    else:
        psnr = E.evaluate_model_single(tr, W, H, n, frames, str(out), IT, VID, save_checkpoint=False,
                                       output_folder=str(out / "frames"), frame_offset=c0)
    tr.release()
    assert CG._marker(d / it) == "PSNR_%f" % psnr
    a, b = A.clip_own_frames(clip, T, V)
    for t in range(a, b):
        CG._same_bytes(res / "output" / ("%05d.png" % t), out / "frames" / ("%05d.png" % t))


def _check_run(res, refs, data, cfg, tmp, seg=False):
    assert sorted(os.listdir(str(res / "output"))) == ["%05d.png" % t for t in range(T)]
    assert sorted(p for p in os.listdir(str(res)) if p != "output") == [A.clip_name(c) for c in PLAN]
    for k, ref in enumerate(refs):
        _check_clip(res, k, ref, data, cfg, tmp, seg)
    _check_seams(res, cfg, seg)


def _stand_alone(tmp_path_factory, data, script, args, name):
    refs = []
    for k, clip in enumerate(PLAN):
        w = tmp_path_factory.mktemp(f"{name}_alone{k}")
        CG._clip_folder(data, w / "data" / "test" / VID, clip)
        _script(script, args, w)
        refs.append(w / "results" / VID / "stage_1")
    return refs


@pytest.fixture(scope="module")
def atlas_run(tmp_path_factory):
    """The atlas script with --clips --clip_overlap 2 on the 15-frame video, and stand-alone on each clip's folder."""
    work = tmp_path_factory.mktemp("overlap_atlas")
    data = work / "data" / "test" / VID
    CG._write_video(data, T)
    cfg, path = CG._config(work, **SMALL)
    args = ["--vid_name", VID, "--root", "data/test/", "--down", "1", "--config", path]
    r = _script("stage1_neural_atlas.py", args + ["--clips", "--clip_overlap", str(V)], work)
    assert "stitch: rank 0 wrote 4 frames of 2 seams in " in r.stdout
    return work, cfg, path, _stand_alone(tmp_path_factory, data, "stage1_neural_atlas.py", args, "atlas")


def test_atlas_script_with_overlap(atlas_run, tmp_path):
    work, cfg, _, refs = atlas_run
    assert A.clip_plan(T, M, V) == PLAN and A.clip_seams(PLAN) == SEAMS
    _check_run(work / "results" / VID / "stage_1", refs, work / "data" / "test" / VID, cfg, tmp_path)


def test_atlas_stitch_under_torchrun_and_emulated_ranks(atlas_run, tmp_path, monkeypatch):
    """The stitch under torch.distributed.run (two ranks when the node has two GPUs), and ranks 0 and 1 of 2 in this
    process, from the one-process run's checkpoints: the same shared frames."""
    from src.models.stage_1 import driver as D
    from src.stage1_neural_atlas import VARIANT
    work, cfg, path, _ = atlas_run
    one = work / "results" / VID / "stage_1"
    nproc = min(2, torch.cuda.device_count())
    run = tmp_path / "torchrun"
    data = run / "data" / "test" / VID
    CG._write_video(data, T)
    _run([sys.executable, "-m", "torch.distributed.run", "--standalone", "--nproc-per-node", str(nproc), WRAPPER,
          str(SEED), os.path.join(PKG, "src", "stage1_neural_atlas.py"), "--vid_name", VID, "--root", "data/test/",
          "--down", "1", "--config", path, "--clips", "--clip_overlap", str(V), "--gpus", str(nproc)], run)
    res = run / "results" / VID / "stage_1"
    assert sorted(os.listdir(str(res / "output"))) == ["%05d.png" % t for t in range(T)]
    _check_seams(res, cfg, False)
    # the same checkpoints give the same shared frames, whichever ranks stitch them
    for c in PLAN:
        CG._close_checkpoint(res / A.clip_name(c) / "checkpoint", one / A.clip_name(c) / "checkpoint")
    emu = tmp_path / "emulated"
    shutil.copytree(str(one), str(emu / "results" / VID / "stage_1"))
    CG._write_video(emu / "data" / "test" / VID, T)
    for t in range(T):
        os.remove(str(emu / "results" / VID / "stage_1" / "output" / ("%05d.png" % t)))
    monkeypatch.chdir(emu)
    args = types.SimpleNamespace(vid_path=str(emu / "data" / "test" / VID), down=1)
    assert [D.stitch(VARIANT, cfg, args, PLAN, DEV, r, 2) for r in range(2)] == [2, 2]
    assert sorted(os.listdir(str(emu / "results" / VID / "stage_1" / "output"))) == \
        ["%05d.png" % t for a, b in SEAMS for t in range(a, b)]
    for a, b in SEAMS:
        for t in range(a, b):
            CG._same_bytes(emu / "results" / VID / "stage_1" / "output" / ("%05d.png" % t), one / "output" / ("%05d.png" % t))


def test_run_without_an_evaluation_stitches_nothing(tmp_path):
    data = tmp_path / "data" / "test" / VID
    CG._write_video(data, T)
    _, path = CG._config(tmp_path, **dict(SMALL, iters_num=2))
    r = _script("stage1_neural_atlas.py", ["--vid_name", VID, "--root", "data/test/", "--down", "1", "--config", path,
                                           "--clips", "--clip_overlap", str(V), "--no_artefacts"], tmp_path)
    assert "nothing was stitched" in r.stdout
    assert glob.glob(str(tmp_path / "results" / VID / "stage_1" / "output" / "*.png")) == []


def test_seg_script_with_overlap(tmp_path_factory, tmp_path):
    work = tmp_path_factory.mktemp("overlap_seg")
    data = work / "data" / "test" / VID
    CG._write_video(data, T)
    cfg, path = CG._config(work, **dict(SMALL, samples_batch=1500))
    args = ["--vid_name", VID, "--root", "data/test/", "--down", "1", "--class_name", "person", "--config", path]
    r = _script("stage1_neural_atlas_seg.py", args + ["--clips", "--clip_overlap", str(V)], work)
    assert "stitch: rank 0 wrote 4 frames of 2 seams in " in r.stdout
    refs = _stand_alone(tmp_path_factory, data, "stage1_neural_atlas_seg.py", args, "seg")
    _check_run(work / "results" / VID / "stage_1", refs, data, cfg, tmp_path, seg=True)


def test_driver_with_overlap_and_flicker_end_to_end(tmp_path):
    from src.models.network_filter import UNet
    from src.models.network_local import TransformNet
    CG._write_video(tmp_path / "data" / "test" / VID, T)
    cfg, path = CG._config(tmp_path, **SMALL)
    pkg = tmp_path / "pkg"
    shutil.copytree(PKG, str(pkg), ignore=shutil.ignore_patterns("__pycache__"))
    shutil.copy(path, str(pkg / "src" / "config" / "config_flow_100.json"))
    os.makedirs(str(tmp_path / "pretrained_weights"))
    torch.manual_seed(0)
    torch.save(UNet(in_channels=6, out_channels=3, init_features=32).state_dict(),
               str(tmp_path / "pretrained_weights" / "neural_filter.pth"))
    tn = TransformNet(types.SimpleNamespace(nf=32, norm="IN", model="TransformNet", blocks=5), nc_in=12, nc_out=3)
    torch.save(tn.state_dict(), str(tmp_path / "pretrained_weights" / "local_refinement_net.pth"))
    env = dict(CG._env(), PYTHONPATH=str(pkg))
    r = subprocess.run([sys.executable, str(pkg / "test.py"), "--video_frame_folder", VID, "--clips", "--clip_overlap",
                        str(V), "--evaluate_flicker"], cwd=str(tmp_path), env=env, capture_output=True, text=True,
                       timeout=1800)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    res = tmp_path / "results" / VID
    assert sorted(p for p in os.listdir(str(res / "stage_1")) if p.startswith("clip_")) == [A.clip_name(c) for c in PLAN]
    for sub in ("stage_1/output", "neural_filter/output", "final/output"):
        assert len(glob.glob(str(res / sub / "*.png"))) == T, sub
    doc = json.load(open(str(res / "flicker.json")))
    assert doc["clips"]["plan"] == [list(c) for c in PLAN]
    # V + 1 = 3 pairs per seam: into the cross-fade, inside it, out of it
    assert doc["clips"]["boundary_pairs"] == [4, 5, 6, 8, 9, 10]
    for s in ("input", "atlas", "final"):
        assert doc["sequences"][s]["E_boundary"] is not None and doc["sequences"][s]["E_interior"] is not None
