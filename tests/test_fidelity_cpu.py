"""The fidelity metric's definition (DESIGN §4f) on its float64 restatement (tests/fidelity_oracle.py), and the host
logic of src/evaluate_flicker.py --fidelity: the JSON document, the frame split and gather over 1 to 4 ranks under
gloo, the clip seam frames and the driver flags.  The kernel is pinned against the same restatement in
tests/test_fidelity_gpu.py."""
import importlib.util
import json
import os
import queue
import socket

import cv2
import numpy as np
import pytest
import torch.distributed as dist
import torch.multiprocessing as mp
from scipy.ndimage import gaussian_filter

import fidelity_oracle as FI
from b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCRIPT = os.path.join(ROOT, "all-in-one-deflicker_b200", "src", "evaluate_flicker.py")


def _script():
    spec = importlib.util.spec_from_file_location("evaluate_flicker", SCRIPT)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_taps_are_scipys_gaussian_weights():
    impulse = np.zeros(21)
    impulse[10] = 1.0
    want = gaussian_filter(impulse, sigma=1.5, truncate=3.5)[5:16]
    assert np.array_equal(FI.taps(), want)
    assert FI.taps().sum() == pytest.approx(1.0, abs=1e-15)


@pytest.mark.parametrize("H,W,Hr,Wr,bits", [(11, 11, 11, 11, 8), (17, 29, 17, 29, 8), (40, 64, 10, 16, 8),
                                            (40, 64, 80, 128, 16), (45, 70, 23, 35, 16)])
def test_restatement_equals_the_plain_scipy_form(H, W, Hr, Wr, bits):
    rng = np.random.default_rng(H * W + Hr)
    o, r = FI.texture(rng, H, W), FI.texture(rng, Hr, Wr, bits)
    got = float(np.nanmean(FI.ssim_map(o, r)))
    assert abs(got - FI.ssim_plain(o, r)) <= 1e-12
    s, _ = FI.frame_values(o, r)
    assert abs(s - got) <= 1e-12


def test_identical_frames_score_one_exactly_and_no_psnr():
    rng = np.random.default_rng(0)
    f = FI.texture(rng, 23, 31)
    smap = FI.ssim_map(f, f)
    assert (smap[5:-5, 5:-5] == 1.0).all() and np.isnan(smap[:5]).all() and np.isnan(smap[:, -5:]).all()
    ssum, sse = FI.frame_sums(f, f)
    assert sse == 0.0 and ssum == 3.0 * 13 * 21
    assert FI.frame_values(f, f) == (1.0, None)


def test_constant_frames_give_the_luminance_term():
    """O = a and R = b everywhere: the variances vanish (to rounding), and SSIM = (2ab + C1) / (a^2 + b^2 + C1)."""
    o = np.full((15, 19, 3), 200, np.uint8)
    r = np.full((15, 19, 3), 60, np.uint8)
    a, b = np.float64(np.float32(200) / np.float32(255)), np.float64(np.float32(60) / np.float32(255))
    want = (2 * a * b + FI.C1) / (a * a + b * b + FI.C1)
    smap = FI.ssim_map(o, r)[5:-5, 5:-5]
    assert np.allclose(smap, want, rtol=1e-12, atol=0)
    _, psnr = FI.frame_values(o, r)
    assert psnr == pytest.approx(10 * np.log10(1 / (a - b) ** 2), rel=1e-12)


def test_global_gain_gives_the_closed_form_per_pixel():
    """O = g R with g = 2 (uint16 values below 2^15: the decoded O is exactly 2 R): mu_O = g mu, var_O = g^2 var,
    cov = g var, with mu and var the local moments of R."""
    rng = np.random.default_rng(1)
    r = (FI.texture(rng, 36, 52, 16) // 2).astype(np.uint16)
    o = (2 * r).astype(np.uint16)
    R = FI.decode(r).astype(np.float64)
    g = 2.0
    f = lambda a: gaussian_filter(a, sigma=1.5, truncate=3.5)
    smap = FI.ssim_map(o, r)
    for c in range(3):
        mu, m2 = f(R[..., c]), f(R[..., c] * R[..., c])
        var = m2 - mu * mu
        want = ((2 * g * mu * mu + FI.C1) * (2 * g * var + FI.C2)) / (((g * g + 1) * mu * mu + FI.C1)
                                                                    * ((g * g + 1) * var + FI.C2))
        assert np.allclose(smap[5:-5, 5:-5, c], want[5:-5, 5:-5], rtol=0, atol=1e-12)


def test_eleven_pixels_give_one_interior_pixel_and_ten_are_refused():
    rng = np.random.default_rng(2)
    o, r = FI.texture(rng, 11, 11), FI.texture(rng, 11, 11)
    smap = FI.ssim_map(o, r)
    inside = ~np.isnan(smap[..., 0])
    assert inside.sum() == 1 and inside[5, 5]
    ssum, _ = FI.frame_sums(o, r)
    assert ssum == (smap[5, 5, 0] + smap[5, 5, 1]) + smap[5, 5, 2]
    for H, W in ((10, 40), (40, 10)):
        with pytest.raises(ValueError, match="11"):
            FI.ssim_map(FI.texture(rng, H, W), FI.texture(rng, H, W))


@pytest.mark.parametrize("scale", [0.25, 2.0])
def test_reference_resize_is_cv2_inter_linear_on_fp32(scale):
    rng = np.random.default_rng(3)
    H, W = 40, 64
    ref = FI.texture(rng, int(H * scale), int(W * scale))
    use = cv2.ipp.useIPP()
    cv2.ipp.setUseIPP(False)                # OpenCV's own code path, which resize_linear.cuh restates
    try:
        want = cv2.resize(FI.decode(ref), (W, H), interpolation=cv2.INTER_LINEAR)
    finally:
        cv2.ipp.setUseIPP(use)
    assert np.array_equal(FI.reference_at(ref, H, W), want)


def test_sixteen_bit_and_eight_bit_scale_to_the_same_values():
    """v / 255 and 257 v / 65535 are the same real number, so an 8-bit frame and its 16-bit copy are identical."""
    rng = np.random.default_rng(4)
    o = FI.texture(rng, 20, 24)
    r = (o.astype(np.uint16) * 257).astype(np.uint16)
    assert np.array_equal(FI.decode(o), FI.decode(r))
    assert FI.frame_values(o, r) == (1.0, None)


# ---------------------------------------------------------------------------------------------------- the script
T_FRAMES = 11


def _write_video(root):
    """data/test/vid (11 frames, 24 x 32, 8-bit), its exact flows, a stage-1 output at 12 x 16 (16-bit), a final output
    at 24 x 32 and a clean reference folder; no filter output."""
    q = synth.quality_set(24, 32, T_FRAMES, seed=5)
    small = synth.quality_set(12, 16, T_FRAMES, seed=6, velocity=(0.75, -0.375))
    dirs = {"input": os.path.join(root, "data", "test", "vid"),
            "atlas": os.path.join(root, "results", "vid", "stage_1", "output"),
            "final": os.path.join(root, "results", "vid", "final", "output"),
            "clean": os.path.join(root, "clean")}
    for d in dirs.values():
        os.makedirs(d)
    flow_dir = dirs["input"] + "_flow"
    os.makedirs(flow_dir)
    u8 = lambda a: np.round(a.numpy() * 255).astype(np.uint8)
    for t in range(T_FRAMES):
        cv2.imwrite(os.path.join(dirs["input"], "%05d.png" % t), u8(q["frames"][..., t]))
        cv2.imwrite(os.path.join(dirs["atlas"], "%05d.png" % t),
                    np.round(small["frames"][..., t].numpy() * 65535).astype(np.uint16))
        cv2.imwrite(os.path.join(dirs["final"], "%05d.png" % t), u8(q["clean"][..., t]))
        cv2.imwrite(os.path.join(dirs["clean"], "%05d.png" % t), u8(q["clean"][..., t]))
    for t in range(T_FRAMES - 1):
        a, b = "%05d.png" % t, "%05d.png" % (t + 1)
        np.save(os.path.join(flow_dir, "%s_%s.npy" % (a, b)), q["flow_fwd"][:, :, :, t, 0].numpy())
        np.save(os.path.join(flow_dir, "%s_%s.npy" % (b, a)), q["flow_bwd"][:, :, :, t + 1, 0].numpy())


def oracle_window(flows, frames):
    """FlickerScorer.score_window on the restatement (tests/flicker_oracle.py)."""
    import flicker_oracle as FO
    return {s: [FO.pair_sums(fr[i], fr[i + 1], *flows[i]) for i in range(min(len(flows), len(fr) - 1))]
            for s, fr in frames.items()}


def oracle_frames(refs, frames):
    """FidelityScorer.score_frames on the restatement."""
    return {s: [FI.frame_sums(f, r) for f, r in zip(fr, refs)] for s, fr in frames.items()}


def _dumps(doc):
    return None if doc is None else json.dumps(doc, indent=1) + "\n"


def _run(root, rank, world, fidelity=True, reference=None, clips=False):
    cwd = os.getcwd()
    os.chdir(root)
    try:
        script = _script()
        if not fidelity:
            return _dumps(script.evaluate("vid", list(script.SEQUENCES), oracle_window, rank, world, clips=clips)), None
        doc, fdoc = script.evaluate_fidelity("vid", list(script.SEQUENCES), oracle_window, oracle_frames, reference,
                                             rank, world, clips=clips)
        return _dumps(doc), _dumps(fdoc)
    finally:
        os.chdir(cwd)


def _worker(rank, world, port, root, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        q.put((rank, _run(root, rank, world, reference="clean")))
        dist.barrier()
    finally:
        dist.destroy_process_group()


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


@pytest.fixture(scope="module")
def video(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("fidelity"))
    _write_video(root)
    return root


def test_single_process_document_against_the_input(video):
    _, raw = _run(video, 0, 1)
    doc = json.loads(raw)
    assert doc["video"] == "vid" and doc["reference"] == os.path.join("data", "test", "vid")
    assert doc["frames"] == T_FRAMES
    seq = doc["sequences"]
    assert list(seq) == ["atlas", "final"]                   # the input is its own reference: not scored
    assert seq["atlas"]["resolution"] == [12, 16] and seq["atlas"]["reference_resolution"] == [24, 32]
    for s in seq.values():
        assert [f["t"] for f in s["per_frame"]] == list(range(T_FRAMES)) and s["identical_frames"] == 0
        assert s["SSIM"] == sum(f["ssim"] for f in s["per_frame"]) / T_FRAMES
        assert s["PSNR"] == sum(f["psnr"] for f in s["per_frame"]) / T_FRAMES


def test_a_separate_reference_scores_the_input_too(video):
    _, raw = _run(video, 0, 1, reference="clean")
    doc = json.loads(raw)
    seq = doc["sequences"]
    assert doc["reference"] == "clean" and list(seq) == ["input", "atlas", "final"]
    # the final output holds the clean frames: identical, S = 1 and PSNR null
    assert seq["final"]["SSIM"] == 1.0 and seq["final"]["PSNR"] is None
    assert seq["final"]["identical_frames"] == T_FRAMES
    assert all(f == {"t": t, "ssim": 1.0, "psnr": None} for t, f in enumerate(seq["final"]["per_frame"]))
    assert seq["input"]["SSIM"] < 1.0 and seq["input"]["PSNR"] > 0
    # per frame, the document holds the restatement's values
    from src.evaluate_flicker import read_frame
    files = sorted(os.listdir(os.path.join(video, "clean")))
    for t in (0, T_FRAMES - 1):
        o = read_frame(os.path.join(video, "data", "test", "vid", files[t]))
        r = read_frame(os.path.join(video, "clean", files[t]))
        assert (seq["input"]["per_frame"][t]["ssim"], seq["input"]["per_frame"][t]["psnr"]) == FI.frame_values(o, r)


def test_flicker_json_is_the_same_with_and_without_fidelity(video):
    plain, _ = _run(video, 0, 1, fidelity=False)
    for reference in (None, "clean"):
        with_fid, _ = _run(video, 0, 1, reference=reference)
        assert with_fid == plain


@pytest.mark.parametrize("world", [2, 3, 4])
def test_frame_split_and_gather_write_the_same_bytes(video, world):
    want = _run(video, 0, 1, reference="clean")
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, video, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = {}
    try:
        for _ in range(world):
            r, out = q.get(timeout=240)
            res[r] = out
    except queue.Empty:
        pass
    for p in procs:
        p.join(timeout=60)
        if p.is_alive():
            p.kill()
    assert sorted(res) == list(range(world)), "a rank did not report"
    assert all(res[r] == (None, None) for r in range(1, world))
    assert res[0] == want


def test_fidelity_alone_reads_no_flows(video, tmp_path):
    """With score_window None only the frames are decoded: the same fidelity document, and no flicker document."""
    import shutil
    root = str(tmp_path / "noflow")
    shutil.copytree(video, root)
    shutil.rmtree(os.path.join(root, "data", "test", "vid_flow"))
    cwd = os.getcwd()
    os.chdir(root)
    try:
        doc, fdoc = _script().evaluate_fidelity("vid", ["atlas", "final"], None, oracle_frames)
    finally:
        os.chdir(cwd)
    assert doc is None and _dumps(fdoc) == _run(video, 0, 1)[1]


def test_seam_frames_of_three_clip_plans():
    script = _script()
    plan, seams = script.clip_seam_frames(500)                 # maximum_number_of_frames = 200
    assert plan == [(0, 167), (167, 334), (334, 500)] and seams == [167, 334]
    plan, seams = script.clip_seam_frames(500, 8)
    from b200.atlas import clip_seams
    assert seams == [t for a, b in clip_seams(plan) for t in range(a, b)] and len(seams) == 16
    assert all(plan[k + 1][0] <= t < plan[k][1] for k, t in zip([0] * 8 + [1] * 8, seams))
    scores = [(3.0 * (0.5 if t in seams else 0.9) * (16 - 10) * (16 - 10), 3.0 * 16 * 16 * 1e-3) for t in range(500)]
    doc = script.report_fidelity("v", 500, "r", (16, 16), {"final": (16, 16)}, {"final": "x"}, {"final": scores},
                                 (plan, seams))
    e = doc["sequences"]["final"]
    assert doc["clips"] == {"plan": [list(c) for c in plan], "seam_frames": seams}
    assert e["SSIM_seam"] == 0.5 and e["SSIM_interior"] == pytest.approx(0.9, rel=1e-15)
    assert e["PSNR_seam"] == pytest.approx(30.0, rel=1e-12) and e["PSNR_interior"] == pytest.approx(30.0, rel=1e-12)
    assert "SSIM_seam" in script.fidelity_table(doc)


def test_script_refuses_reference_without_fidelity():
    with pytest.raises(SystemExit) as e:
        _script().main(["--video_name", "v", "--reference", "clean"])
    assert e.value.code == 2


def test_driver_passes_the_flags_on_and_refuses_fidelity_alone(tmp_path, monkeypatch):
    import runpy
    import subprocess
    import sys
    os.makedirs(str(tmp_path / "data" / "test" / "long"))
    monkeypatch.chdir(tmp_path)
    calls = []
    monkeypatch.setattr(subprocess, "call", lambda cmd, *a, **k: calls.append(list(cmd)) or 0)
    pkg = os.path.join(ROOT, "all-in-one-deflicker_b200")
    run = lambda extra: runpy.run_path(os.path.join(pkg, "test.py"), run_name="__main__")
    for extra in (["--evaluate_flicker"], ["--evaluate_flicker", "--fidelity"],
                  ["--evaluate_flicker", "--fidelity", "--reference", "clean", "--clips"]):
        calls.clear()
        monkeypatch.setattr(sys, "argv", ["test.py", "--video_frame_folder", "long"] + extra)
        with pytest.raises(SystemExit) as e:
            run(extra)
        assert e.value.code == 0
        stage1, stage2, flicker = calls
        assert "--fidelity" not in stage1 + stage2 and "--reference" not in stage1 + stage2
        assert ("--fidelity" in flicker) == ("--fidelity" in extra)
        if "--reference" in extra:
            assert flicker[flicker.index("--reference") + 1] == "clean"
        else:
            assert "--reference" not in flicker
    for extra in (["--fidelity"], ["--evaluate_flicker", "--reference", "clean"]):
        calls.clear()
        monkeypatch.setattr(sys, "argv", ["test.py", "--video_frame_folder", "long"] + extra)
        with pytest.raises(SystemExit) as e:
            run(extra)
        assert e.value.code == 2 and not calls


def test_entry_point_validates_its_arguments():
    """Host-side checks of b200_fidelity (no device work: the pointers below are never dereferenced)."""
    import ctypes as C
    from b200 import _native as N
    from csrc_build import ensure_built
    ensure_built()
    lib = N.lib()
    good = N.FidelityFrame(0x1000, 0x2000, 1080, 1920, 270, 480, 8, 16)
    table = lambda *d: (N.FidelityFrame * len(d))(*d)
    one = int(lib.b200_fidelity_workspace_bytes(table(good), 1))
    # the partials: two doubles per 16 x 32 tile
    assert one == 2 * (1080 // 16 + 1) * (1920 // 32) * 8
    small = N.FidelityFrame(0x1000, 0x2000, 11, 11, 1, 1, 16, 8)
    assert lib.b200_fidelity_workspace_bytes(table(small), 1) == 2 * 8
    assert lib.b200_fidelity_workspace_bytes(table(good, small), 2) == one + 2 * 8
    cases = [
        (N.FidelityFrame(0, 0x2000, 16, 16, 16, 16, 8, 8), b"null pointer"),
        (N.FidelityFrame(0x1000, 0, 16, 16, 16, 16, 8, 8), b"null pointer"),
        (N.FidelityFrame(0x1000, 0x2000, 10, 16, 16, 16, 8, 8), b"11 x 11"),
        (N.FidelityFrame(0x1000, 0x2000, 16, 10, 16, 16, 8, 8), b"11 x 11"),
        (N.FidelityFrame(0x1000, 0x2000, 40000, 16, 16, 16, 8, 8), b"11 x 11"),
        (N.FidelityFrame(0x1000, 0x2000, 16, 16, 0, 16, 8, 8), b"reference 0 x 16"),
        (N.FidelityFrame(0x1000, 0x2000, 16, 16, 16, 40000, 8, 8), b"reference"),
        (N.FidelityFrame(0x1000, 0x2000, 16, 16, 16, 16, 12, 8), b"12 and 8 bits"),
        (N.FidelityFrame(0x1000, 0x2000, 16, 16, 16, 16, 8, 10), b"8 and 10 bits"),
        (N.FidelityFrame(0x1001, 0x2000, 16, 16, 16, 16, 16, 8), b"aligned"),
        (N.FidelityFrame(0x1000, 0x2001, 16, 16, 16, 16, 8, 16), b"aligned"),
    ]
    for bad, msg in cases:
        assert lib.b200_fidelity_workspace_bytes(table(good, bad), 2) == -1
        assert msg in lib.b200_last_error() and b"frame 1" in lib.b200_last_error()
    # odd addresses are fine for 8-bit frames
    assert lib.b200_fidelity_workspace_bytes(table(N.FidelityFrame(0x1001, 0x2001, 16, 16, 16, 16, 8, 8)), 1) > 0
    assert lib.b200_fidelity_workspace_bytes(table(good), 0) == -1 and b"1 to 32" in lib.b200_last_error()
    assert lib.b200_fidelity_workspace_bytes(table(*[good] * 33), 33) == -1
    assert lib.b200_fidelity_workspace_bytes(None, 1) == -1
    sums, ws = C.c_void_p(0x5000), C.c_void_p(0x6000)
    assert lib.b200_fidelity(table(good), 1, sums, None, ws, one - 8, None) == 3       # B200_ERR_WORKSPACE
    assert b"need %d bytes" % one in lib.b200_last_error()
    assert lib.b200_fidelity(table(good), 1, None, None, ws, one, None) == 1
    assert lib.b200_fidelity(table(good), 1, sums, None, C.c_void_p(0x6004), one, None) == 1
