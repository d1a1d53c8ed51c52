"""b200_fidelity (csrc/fidelity.cu) against the float64 restatement of tests/fidelity_oracle.py, and
src/evaluate_flicker.py --fidelity end to end (DESIGN §4f).

The kernel computes in float64 in the restatement's operation order and rounds each pixel's SSIM to fp32 once, so
    |map - restated| <= 2^-24 |restated|            (one rounding to nearest)
with NaN at the same places (outside the interior), and the sums equal the restatement's float64 sums in the kernel's
order bit for bit.  They do not change between calls, graph replays and batch compositions."""
import json
import os
import subprocess
import sys

import cv2
import numpy as np
import pytest
import torch

import fidelity_oracle as FI
from b200 import fidelity as FD
from b200 import synth

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "all-in-one-deflicker_b200")
DEV = torch.device("cuda:0")
REL = 2.0 ** -24


def _case(seed, H, W, Hr=None, Wr=None, bits=8, ref_bits=8, related=True):
    """A frame and a reference: the reference is a noisy copy of the frame's content (so SSIM spans its range) or,
    with related=False, independent."""
    rng = np.random.default_rng(seed)
    Hr, Wr = Hr or H, Wr or W
    o = FI.texture(rng, H, W, bits)
    if not related:
        return o, FI.texture(rng, Hr, Wr, ref_bits)
    top = 255 if ref_bits == 8 else 65535
    base = cv2.resize(FI.decode(o), (Wr, Hr), interpolation=cv2.INTER_LINEAR).reshape(Hr, Wr, 3)
    r = np.clip(base + 0.08 * rng.standard_normal((Hr, Wr, 3)), 0, 1)
    return o, np.round(r * top).astype(np.uint8 if ref_bits == 8 else np.uint16)


CASES = {
    "11x11": _case(1, 11, 11, related=False),
    "17x29": _case(2, 17, 29),
    "270x480": _case(3, 270, 480),
    "272x480_ref_quarter": _case(4, 272, 480, 68, 120),
    "270x480_16bit_ref_double": _case(5, 270, 480, 540, 960, bits=16),
    "270x480_ref_16bit_half": _case(6, 270, 480, 135, 240, ref_bits=16),
    "1080x1920": _case(7, 1080, 1920),
    "1080x1920_16bit_ref_half": _case(8, 1080, 1920, 540, 960, bits=16, ref_bits=16),
}
_same = FI.texture(np.random.default_rng(9), 40, 64)
CASES["identical"] = (_same, _same.copy())


def _dev(case):
    return [torch.from_numpy(np.ascontiguousarray(a)).to(DEV) for a in case]


def _run(cases, maps=True):
    """One b200_fidelity call on `cases` (lists of device tensors): sums (n, 2) and per-pixel maps, per frame."""
    descs = [FD.frame_desc(*c) for c in cases]
    ws = torch.empty(FD.workspace_bytes(descs), dtype=torch.uint8, device=DEV)
    sums = torch.full((len(cases), 2), float("nan"), dtype=torch.float64, device=DEV)
    px = [c[0].shape[0] * c[0].shape[1] * 3 for c in cases]
    smap = torch.full((sum(px),), 7.0, device=DEV) if maps else None
    FD.fidelity(descs, sums, ws, smap)
    torch.cuda.synchronize()
    out, o = [], 0
    for c, n in zip(cases, px):
        out.append(smap[o:o + n].view(c[0].shape).cpu().numpy() if maps else None)
        o += n
    return sums.cpu().numpy(), out


@pytest.fixture(scope="module")
def batch():
    names = list(CASES)
    dev = {k: _dev(CASES[k]) for k in names}
    sums, maps = _run([dev[k] for k in names])
    return names, dev, sums, maps


@pytest.mark.parametrize("name", list(CASES))
def test_map_and_sums_against_the_restatement(batch, name):
    names, _, sums, maps = batch
    i = names.index(name)
    o, r = CASES[name]
    ref = FI.ssim_map(o, r)
    got = maps[i].astype(np.float64)
    assert (np.isnan(got) == np.isnan(ref)).all()
    inside = ~np.isnan(ref)
    worst = np.abs(got[inside] - ref[inside]).max()
    print(f"{name}: SSIM {np.mean(ref[inside]):.6f}, map max |error| {worst:.3g}")
    assert (np.abs(got[inside] - ref[inside]) <= REL * np.abs(ref[inside])).all()
    want = FI.frame_sums(o, r, ref)
    assert (sums[i, 0], sums[i, 1]) == want
    if name == "identical":
        assert sums[i, 1] == 0 and FD.frame_values(*sums[i], *o.shape[:2]) == (1.0, None)
    else:
        assert sums[i, 1] > 0


def test_bit_identity_over_calls_graph_replays_and_batches(batch):
    names, dev, sums, _ = batch
    again, _ = _run([dev[k] for k in names], maps=False)
    assert again.tobytes() == sums.tobytes()
    singles = np.concatenate([_run([dev[k]], maps=False)[0] for k in names])
    assert singles.tobytes() == sums.tobytes()
    rev, _ = _run([dev[k] for k in reversed(names)], maps=False)
    assert rev[::-1].tobytes() == sums.tobytes()
    descs = [FD.frame_desc(*dev[k]) for k in names]
    ws = torch.empty(FD.workspace_bytes(descs), dtype=torch.uint8, device=DEV)
    out = torch.zeros(len(names), 2, dtype=torch.float64, device=DEV)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        FD.fidelity(descs, out, ws)                     # warm up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        FD.fidelity(descs, out, ws)
    for _ in range(2):
        out.zero_()
        g.replay()
        torch.cuda.synchronize()
        assert out.cpu().numpy().tobytes() == sums.tobytes()


def test_scorer_windows_equal_single_calls():
    """FidelityScorer.score_frames: three sequences (8-bit, 16-bit, a lower resolution) against a window of 12
    references (36 frames: two calls), one of them shorter than the window."""
    rng = np.random.default_rng(11)
    H, W = 90, 160
    refs = [FI.texture(rng, H, W) for _ in range(12)]
    frames = {"a": [FI.texture(rng, H, W) for _ in range(12)], "b": [FI.texture(rng, H, W, 16) for _ in range(12)],
              "c": [FI.texture(rng, 45, 80) for _ in range(9)]}
    got = FD.FidelityScorer(DEV).score_frames(refs, frames)
    assert [len(got[k]) for k in "abc"] == [12, 12, 9]
    for k, fr in frames.items():
        for i, v in enumerate(got[k]):
            s, _ = _run([_dev((fr[i], refs[i]))], maps=False)
            assert v == (s[0, 0], s[0, 1])


# ------------------------------------------------------------------------------------------------- end to end
QH, QW, QT = 432, 768, 80
FIXTURE = os.path.join(ROOT, "tests", "golden", "quality_oracle.npz")
# measured on an NVIDIA H100 80GB HBM3 at 700 W (DESIGN §4f) against the clean frames: SSIM of the flickering input
# 0.98907 (1 - SSIM = 0.0109), of the render of the trained parameters 0.99363 (1 - SSIM = 0.0064); the bounds are
# about twice those distances from 1 (the render with two channels exchanged scores about 0.913)
MIN_INPUT_SSIM = 1 - 0.022
MIN_RENDER_SSIM = 1 - 0.013


def _score(root, *extra):
    env = dict(os.environ, PYTHONPATH=PKG)
    for k in ("WORLD_SIZE", "RANK", "LOCAL_RANK"):
        env.pop(k, None)
    r = subprocess.run([sys.executable, os.path.join(PKG, "src", "evaluate_flicker.py"), "--video_name", "q"] + list(extra),
                       cwd=root, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    print(r.stdout)
    out = {}
    for f in ("flicker.json", "fidelity.json"):
        p = os.path.join(root, "results", "q", f)
        if os.path.exists(p):
            with open(p, "rb") as fh:
                out[f] = fh.read()
            if f == "fidelity.json":
                os.remove(p)
    return out


def _unflat(spec, flat):
    from oracle import atlas_oracle as O
    out, off = [], 0
    for k, n in spec.layer_dims():
        out += [torch.from_numpy(flat[off:off + k * n]).view(n, k)]
        off += k * n
        out += [torch.from_numpy(flat[off:off + n])]
        off += n
    return O.state_dict_of(out)


def _write_quality_video(root):
    """The quality set's flickering frames as the input, with their exact flows; the render of quality_oracle.npz's
    trained parameters as the atlas output; the clean frames as the final output and as the reference folder `clean`.
    Every folder holds the set's channels in one order: the parameters were fitted to q["frames"] as they are, so the
    render is written as it comes, like the frames."""
    from b200 import _native as N
    from b200 import atlas as A
    from oracle import atlas_oracle as O
    q = synth.quality_set(QH, QW, QT, seed=0)
    dirs = {"input": os.path.join(root, "data", "test", "q"),
            "atlas": os.path.join(root, "results", "q", "stage_1", "output"),
            "final": os.path.join(root, "results", "q", "final", "output"),
            "clean": os.path.join(root, "clean")}
    for d in dirs.values():
        os.makedirs(d)
    os.makedirs(dirs["input"] + "_flow")
    u8 = lambda a: np.round(np.clip(a, 0, 1) * 255).astype(np.uint8)
    for t in range(QT):
        cv2.imwrite(os.path.join(dirs["input"], "%05d.png" % t), u8(q["frames"][..., t].numpy()))
        for k in ("final", "clean"):
            cv2.imwrite(os.path.join(dirs[k], "%05d.png" % t), u8(q["clean"][..., t].numpy()))
    for t in range(QT - 1):
        a, b = "%05d.png" % t, "%05d.png" % (t + 1)
        np.save(os.path.join(dirs["input"] + "_flow", "%s_%s.npy" % (a, b)), q["flow_fwd"][:, :, :, t, 0].numpy())
        np.save(os.path.join(dirs["input"] + "_flow", "%s_%s.npy" % (b, a)), q["flow_bwd"][:, :, :, t + 1, 0].numpy())
    fx = np.load(FIXTURE)
    assert tuple(int(v) for v in fx["video"]) == (QT, QH, QW)
    tr = A.AtlasTrainer(None, precision=N.PREC_TC, device=DEV)
    tr.load_state(_unflat(O.MAPPING_SPEC, fx["mapping_params"]), _unflat(O.ATLAS_SPEC, fx["atlas_params"]))
    for t in range(QT):
        _, rgb = tr.render_frame(t, QH, QW, QT, want_u8=True)
        cv2.imwrite(os.path.join(dirs["atlas"], "%05d.png" % t), rgb.cpu().numpy())


@pytest.fixture(scope="module")
def quality_run(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("fidelity_e2e"))
    _write_quality_video(root)
    plain = _score(root)
    fid = _score(root, "--fidelity", "--reference", "clean")
    return root, plain, fid


def test_quality_set_end_to_end(quality_run):
    _, plain, fid = quality_run
    assert "fidelity.json" not in plain
    assert fid["flicker.json"] == plain["flicker.json"]
    doc = json.loads(fid["fidelity.json"])
    seq = doc["sequences"]
    assert doc["reference"] == "clean" and doc["frames"] == QT
    assert list(seq) == ["input", "atlas", "final"]
    for s in seq.values():
        assert len(s["per_frame"]) == QT and s["reference_resolution"] == [QH, QW]
        assert s["SSIM"] == sum(f["ssim"] for f in s["per_frame"]) / QT
    print({k: (v["SSIM"], v["PSNR"]) for k, v in seq.items()})
    # the final folder holds the clean frames themselves
    assert seq["final"]["SSIM"] == 1.0 and seq["final"]["PSNR"] is None and seq["final"]["identical_frames"] == QT
    assert seq["input"]["identical_frames"] == 0 and seq["input"]["SSIM"] > MIN_INPUT_SSIM
    assert seq["atlas"]["SSIM"] > MIN_RENDER_SSIM


def test_render_and_reference_share_the_channel_order(quality_run):
    """SSIM and PSNR compare channel by channel: the render scores higher against the clean frames as written than
    with its first and last channels exchanged."""
    root, _, _ = quality_run
    from src.evaluate_flicker import read_frame
    a = read_frame(os.path.join(root, "results", "q", "stage_1", "output", "00040.png"))
    c = read_frame(os.path.join(root, "clean", "00040.png"))
    same, swapped = FI.frame_values(a, c), FI.frame_values(np.ascontiguousarray(a[..., ::-1]), c)
    print("frame 40 against the clean frame: as written %s, channels exchanged %s" % (same, swapped))
    assert same[0] > swapped[0] and same[1] > swapped[1]


def test_script_frames_equal_the_restatement(quality_run):
    root, _, fid = quality_run
    doc = json.loads(fid["fidelity.json"])
    from src.evaluate_flicker import frame_files, read_frame
    refs = frame_files(os.path.join(root, "clean"))
    for s, entry in doc["sequences"].items():
        files = frame_files(os.path.join(root, entry["folder"]))
        for t in (0, 41, QT - 1):
            want = FI.frame_values(read_frame(files[t]), read_frame(refs[t]))
            assert (entry["per_frame"][t]["ssim"], entry["per_frame"][t]["psnr"]) == want, (s, t)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_two_gpus_write_the_same_bytes(quality_run):
    root, _, fid = quality_run
    assert _score(root, "--fidelity", "--reference", "clean", "--gpus", "2") == fid


def test_driver_with_evaluate_flicker_and_fidelity(tmp_path):
    """test.py --evaluate_flicker --fidelity on a 13-frame 96 x 128 video with exact flows: stage 1 (a short fit),
    stage 2 (random weights), the warping error and the fidelity of the three outputs to the input."""
    import shutil
    import types
    from src.models.network_filter import UNet
    from src.models.network_local import TransformNet
    q = synth.quality_set(96, 128, 13, seed=2)
    vid = tmp_path / "data" / "test" / "v"
    os.makedirs(str(vid) + "_flow")
    os.makedirs(str(vid))
    for t in range(13):
        cv2.imwrite(str(vid / ("%05d.png" % t)), np.round(q["frames"][..., t].numpy() * 255).astype(np.uint8))
    for t in range(12):
        a, b = "%05d.png" % t, "%05d.png" % (t + 1)
        np.save(str(vid) + "_flow/%s_%s.npy" % (a, b), q["flow_fwd"][:, :, :, t, 0].numpy())
        np.save(str(vid) + "_flow/%s_%s.npy" % (b, a), q["flow_bwd"][:, :, :, t + 1, 0].numpy())
    cfg = json.load(open(os.path.join(PKG, "src", "config", "config_flow_100.json")))
    cfg.update(maximum_number_of_frames=13, iters_num=21, evaluate_every=20, pretrain_iter_number=2, samples_batch=2000,
               stop_global_rigidity=10)
    pkg = tmp_path / "pkg"
    shutil.copytree(PKG, str(pkg), ignore=shutil.ignore_patterns("__pycache__"))
    json.dump(cfg, open(str(pkg / "src" / "config" / "config_flow_100.json"), "w"))
    os.makedirs(str(tmp_path / "pretrained_weights"))
    torch.manual_seed(0)
    torch.save(UNet(in_channels=6, out_channels=3, init_features=32).state_dict(),
               str(tmp_path / "pretrained_weights" / "neural_filter.pth"))
    tn = TransformNet(types.SimpleNamespace(nf=32, norm="IN", model="TransformNet", blocks=5), nc_in=12, nc_out=3)
    torch.save(tn.state_dict(), str(tmp_path / "pretrained_weights" / "local_refinement_net.pth"))
    env = dict(os.environ, PYTHONPATH=str(pkg), B200_ALLOW_RANDOM_RAFT="1")
    for k in ("WORLD_SIZE", "RANK", "LOCAL_RANK"):
        env.pop(k, None)
    r = subprocess.run([sys.executable, str(pkg / "test.py"), "--video_frame_folder", "v", "--evaluate_flicker",
                        "--fidelity"], cwd=str(tmp_path), env=env, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    print(r.stdout[-1500:])
    flick = json.load(open(str(tmp_path / "results" / "v" / "flicker.json")))
    doc = json.load(open(str(tmp_path / "results" / "v" / "fidelity.json")))
    assert list(flick["sequences"]) == ["input", "atlas", "filter", "final"]
    assert list(doc["sequences"]) == ["atlas", "filter", "final"] and doc["frames"] == 13
    for s in doc["sequences"].values():
        assert len(s["per_frame"]) == 13 and -1 <= s["SSIM"] <= 1 and s["PSNR"] is not None
