"""The temporal warping error's definition (DESIGN §4e) on its float64 restatement (tests/flicker_oracle.py), and the
host logic of src/evaluate_flicker.py: the JSON document, the pair split and gather over 1 to 4 ranks under gloo, and
the clip-boundary pairs.  The kernel is pinned against the same restatement in tests/test_flicker_gpu.py."""
import importlib.util
import json
import math
import os
import queue
import socket

import cv2
import numpy as np
import pytest
import torch.distributed as dist
import torch.multiprocessing as mp

import flicker_oracle as FO
from b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCRIPT = os.path.join(ROOT, "all-in-one-deflicker_b200", "src", "evaluate_flicker.py")


def _script():
    spec = importlib.util.spec_from_file_location("evaluate_flicker", SCRIPT)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _const_flow(H, W, vx, vy):
    f = np.empty((H, W, 2), np.float32)
    f[..., 0], f[..., 1] = vx, vy
    return f


def _inside(H, W, vx, vy):
    yy, xx = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    return (xx + vx >= 0) & (xx + vx <= W - 1) & (yy + vy >= 0) & (yy + vy <= H - 1)


def test_identical_frames_with_zero_flow_score_zero():
    rng = np.random.default_rng(0)
    f = rng.integers(0, 256, (17, 23, 3), dtype=np.uint8)
    z = np.zeros((17, 23, 2), np.float32)
    err, mask = FO.warp_maps(f, f, z, z)
    assert mask.all() and not err.any()
    assert FO.pair_value(f, f, z, z) == 0.0


def test_global_gain_on_exact_flows_gives_the_closed_form():
    """Frame t+1 = g x frame t moved by the quality set's exact integer flow: on every pixel of the mask the error is
    (g - 1)^2 sum_c O_t^2 exactly (uint16 values below 2^15, g = 2: the decoded frame t+1 is exactly 2 O_t)."""
    H, W, v = 40, 56, (2.0, -1.0)
    clean = synth.quality_set(H, W, 2, seed=3, velocity=v)["clean"].numpy()
    u0 = np.round(clean[..., 0] * 32767).astype(np.uint16)
    u1 = (2 * np.round(clean[..., 1] * 32767)).astype(np.uint16)
    fwd, bwd = _const_flow(H, W, *v), _const_flow(H, W, -v[0], -v[1])
    err, mask = FO.warp_maps(u0, u1, fwd, bwd)
    assert (mask == _inside(H, W, *v)).all()
    o = FO.decode(u0)
    want = (2.0 - 1.0) ** 2 * np.sum((o * o).sum(axis=2)[mask]) / (3 * mask.sum())
    assert FO.pair_value(u0, u1, fwd, bwd) == pytest.approx(want, rel=1e-6)
    # the flickering frames of the set score above their clean frames on the same flows
    q = synth.quality_set(H, W, 2, seed=3, velocity=v)
    u8 = lambda a: np.round(a * 255).astype(np.uint8)
    flick = FO.pair_value(u8(q["frames"].numpy()[..., 0]), u8(q["frames"].numpy()[..., 1]), fwd, bwd)
    steady = FO.pair_value(u8(clean[..., 0]), u8(clean[..., 1]), fwd, bwd)
    assert steady < 1e-5 < flick


def test_opposite_exact_flows_keep_every_in_frame_pixel():
    H, W, v = 33, 47, (1.5, -0.75)
    rng = np.random.default_rng(1)
    f0, f1 = (rng.integers(0, 256, (H, W, 3), dtype=np.uint8) for _ in range(2))
    _, mask = FO.warp_maps(f0, f1, _const_flow(H, W, *v), _const_flow(H, W, -v[0], -v[1]))
    assert (mask == _inside(H, W, *v)).all() and mask.sum() == (W - 2) * (H - 1)


def test_occluding_patch_is_excluded():
    """B disagrees with F on a patch: the pixels whose four taps of B all lie in it leave the mask, the pixels whose
    taps all lie outside it stay."""
    H, W, v = 30, 40, (1.5, 0.5)
    f = np.full((H, W, 3), 128, np.uint8)
    fwd, bwd = _const_flow(H, W, *v), _const_flow(H, W, -v[0], -v[1])
    bwd[10:20, 15:25] = (6.0, -3.0)
    _, mask = FO.warp_maps(f, f, fwd, bwd)
    yy, xx = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    qx, qy = xx + v[0], yy + v[1]
    x0, y0 = np.floor(qx), np.floor(qy)
    in_patch = (x0 >= 15) & (x0 + 1 <= 24) & (y0 >= 10) & (y0 + 1 <= 19)
    off_patch = (x0 + 1 < 15) | (x0 > 24) | (y0 + 1 < 10) | (y0 > 19)
    inside = _inside(H, W, *v)
    assert in_patch.sum() > 0 and not mask[in_patch].any()
    assert mask[off_patch & inside].all()


def test_flow_leaving_the_frame_gives_an_empty_pair():
    H, W = 12, 16
    f = np.zeros((H, W, 3), np.uint8)
    fwd, bwd = _const_flow(H, W, W + 3.0, 0.0), _const_flow(H, W, 0.0, 0.0)
    _, mask = FO.warp_maps(f, f, fwd, bwd)
    assert not mask.any() and math.isnan(FO.pair_value(f, f, fwd, bwd))
    doc = _script().report("v", 1, {"input": (H, W)}, {"input": "x"}, {"input": [(0.0, 0.0)]})
    e = doc["sequences"]["input"]
    assert e["per_pair"] == [{"t": 0, "E": None, "mask": 0}] and e["E_warp"] is None and e["empty_pairs"] == 1


def test_flow_resize_scales_x_by_the_width_ratio_and_y_by_the_height_ratio():
    """Frames 16 x 48 whose content moves (+4, +2) pixels; flows at 32 x 24 (twice the height, half the width) hold
    (2, 4).  Scaled geometrically they become (4, 2) and the pair scores 0; resize_flow's swapped factors would give
    (1, 8)."""
    H, W = 16, 48
    rng = np.random.default_rng(2)
    big = rng.integers(0, 256, (H + 8, W + 8, 3), dtype=np.uint8)
    f0, f1 = big[4:4 + H, 4:4 + W].copy(), big[2:2 + H, 0:W].copy()
    fwd, bwd = _const_flow(32, 24, 2.0, 4.0), _const_flow(32, 24, -2.0, -4.0)
    r = FO.resize_flow(fwd, H, W)
    assert np.allclose(r[..., 0], 4.0, rtol=0, atol=1e-6) and np.allclose(r[..., 1], 2.0, rtol=0, atol=1e-6)
    err, mask = FO.warp_maps(f0, f1, fwd, bwd)
    assert mask.sum() == (W - 4) * (H - 2) and np.abs(err[mask]).max() < 1e-9
    swapped = _const_flow(H, W, 1.0, 8.0)
    assert FO.pair_value(f0, f1, swapped, -swapped) > 1e-3


# ---------------------------------------------------------------------------------------------------- the script
T_FRAMES = 11


def _write_video(root):
    """data/test/vid (11 frames, 20 x 28, 8-bit), its exact flows, a stage-1 output at 10 x 14 (16-bit) and a final
    output at 20 x 28; no filter output."""
    q = synth.quality_set(20, 28, T_FRAMES, seed=5)
    small = synth.quality_set(10, 14, T_FRAMES, seed=6, velocity=(0.75, -0.375))
    dirs = {"input": os.path.join(root, "data", "test", "vid"),
            "atlas": os.path.join(root, "results", "vid", "stage_1", "output"),
            "final": os.path.join(root, "results", "vid", "final", "output")}
    for d in dirs.values():
        os.makedirs(d)
    flow_dir = dirs["input"] + "_flow"
    os.makedirs(flow_dir)
    for t in range(T_FRAMES):
        cv2.imwrite(os.path.join(dirs["input"], "%05d.png" % t), np.round(q["frames"][..., t].numpy() * 255).astype(np.uint8))
        cv2.imwrite(os.path.join(dirs["atlas"], "%05d.png" % t),
                    np.round(small["frames"][..., t].numpy() * 65535).astype(np.uint16))
        cv2.imwrite(os.path.join(dirs["final"], "%05d.png" % t), np.round(q["clean"][..., t].numpy() * 255).astype(np.uint8))
    for t in range(T_FRAMES - 1):
        a, b = "%05d.png" % t, "%05d.png" % (t + 1)
        np.save(os.path.join(flow_dir, "%s_%s.npy" % (a, b)), q["flow_fwd"][:, :, :, t, 0].numpy())
        np.save(os.path.join(flow_dir, "%s_%s.npy" % (b, a)), q["flow_bwd"][:, :, :, t + 1, 0].numpy())


def oracle_window(flows, frames):
    """FlickerScorer.score_window on the restatement."""
    return {s: [FO.pair_sums(fr[i], fr[i + 1], *flows[i]) for i in range(min(len(flows), len(fr) - 1))]
            for s, fr in frames.items()}


def _run(root, rank, world, clips=False):
    cwd = os.getcwd()
    os.chdir(root)
    try:
        script = _script()
        doc = script.evaluate("vid", list(script.SEQUENCES), oracle_window, rank, world, clips=clips)
        return None if doc is None else json.dumps(doc, indent=1) + "\n"
    finally:
        os.chdir(cwd)


def _worker(rank, world, port, root, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        q.put((rank, _run(root, rank, world)))
        dist.barrier()
    finally:
        dist.destroy_process_group()


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


@pytest.fixture(scope="module")
def video(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("flicker"))
    _write_video(root)
    return root


def test_single_process_document(video):
    doc = json.loads(_run(video, 0, 1))
    seq = doc["sequences"]
    assert list(seq) == ["input", "atlas", "final"] and doc["pairs"] == T_FRAMES - 1
    assert seq["input"]["resolution"] == [20, 28] and seq["atlas"]["resolution"] == [10, 14]
    for s in seq.values():
        assert [p["t"] for p in s["per_pair"]] == list(range(T_FRAMES - 1)) and s["empty_pairs"] == 0
        assert s["E_warp"] == pytest.approx(np.mean([p["E"] for p in s["per_pair"]]), rel=1e-12)
    # exact flows: the clean frames barely change along them, the flickering input does
    assert seq["final"]["E_warp"] < 0.1 * seq["input"]["E_warp"]
    # every in-frame pixel of the exact flows is in the mask (|v| = (1.5, 0.75))
    assert all(p["mask"] == 26 * 19 for p in seq["input"]["per_pair"])


@pytest.mark.parametrize("world", [2, 3, 4])
def test_pair_split_and_gather_write_the_same_bytes(video, world):
    want = _run(video, 0, 1)
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
    assert all(res[r] is None for r in range(1, world))
    assert res[0] == want


def test_clip_boundary_pairs_of_a_three_clip_plan():
    script = _script()
    plan, boundary = script.clip_boundaries(500)                 # maximum_number_of_frames = 200
    assert plan == [(0, 167), (167, 334), (334, 500)] and boundary == [166, 333]
    scores = [(3.0 * (10.0 if t in boundary else 1.0), 1.0) for t in range(499)]
    doc = script.report("v", 499, {"final": (4, 4)}, {"final": "x"}, {"final": scores}, (plan, boundary))
    e = doc["sequences"]["final"]
    assert doc["clips"] == {"plan": [[0, 167], [167, 334], [334, 500]], "boundary_pairs": [166, 333]}
    assert e["E_boundary"] == 10.0 and e["E_interior"] == 1.0
    assert "E_boundary" in script.table(doc)


def test_kernel_order_sum_is_a_sum():
    rng = np.random.default_rng(4)
    for n in (1, 17 * 5, 256 * 1024 + 3, 1920 * 1080):
        v = rng.random(n)
        assert FO.kernel_order_sum(v) == pytest.approx(float(np.sum(v)), rel=1e-12)


def test_driver_runs_the_score_after_stage2_only_when_asked(tmp_path, monkeypatch):
    import runpy
    import subprocess
    import sys
    os.makedirs(str(tmp_path / "data" / "test" / "long"))
    monkeypatch.chdir(tmp_path)
    calls = []
    monkeypatch.setattr(subprocess, "call", lambda cmd, *a, **k: calls.append(list(cmd)) or 0)
    pkg = os.path.join(ROOT, "all-in-one-deflicker_b200")
    for extra in ([], ["--evaluate_flicker"], ["--evaluate_flicker", "--clips", "--gpus", "2"]):
        calls.clear()
        monkeypatch.setattr(sys, "argv", ["test.py", "--video_frame_folder", "long"] + extra)
        with pytest.raises(SystemExit) as e:
            runpy.run_path(os.path.join(pkg, "test.py"), run_name="__main__")
        assert e.value.code == 0
        if "--evaluate_flicker" not in extra:
            assert len(calls) == 2
            continue
        stage1, stage2, flicker = calls
        assert flicker[1].endswith("evaluate_flicker.py") and flicker[2:4] == ["--video_name", "long"]
        assert ("--clips" in flicker) == ("--clips" in extra) and ("--gpus" in flicker) == ("--gpus" in extra)


def test_entry_point_validates_its_arguments():
    """Host-side checks of b200_warp_error (no device work: the pointers below are never dereferenced)."""
    import ctypes as C
    from b200 import _native as N
    from csrc_build import ensure_built
    ensure_built()
    lib = N.lib()
    good = N.WarpPair(0x1000, 0x2000, 0x3000, 0x4000, 1080, 1920, 540, 960, 8, 0)
    table = lambda *d: (N.WarpPair * len(d))(*d)
    one = int(lib.b200_warp_error_workspace_bytes(table(good), 1))
    # the resized F and B (1080 x 1920 x 2 fp32 each, 256-byte aligned), then 1024 partials of each sum
    assert one == 2 * 1080 * 1920 * 8 + 2 * 1024 * 8
    same = N.WarpPair(0x1000, 0x2000, 0x3000, 0x4000, 17, 5, 17, 5, 16, 0)
    assert lib.b200_warp_error_workspace_bytes(table(same), 1) == 2 * 1 * 8
    cases = [
        (N.WarpPair(0, 0x2000, 0x3000, 0x4000, 4, 4, 4, 4, 8, 0), b"null pointer"),
        (N.WarpPair(0x1000, 0x2000, 0x3000, 0x4000, 0, 4, 4, 4, 8, 0), b"each side"),
        (N.WarpPair(0x1000, 0x2000, 0x3000, 0x4000, 4, 4, 4, 40000, 8, 0), b"each side"),
        (N.WarpPair(0x1000, 0x2000, 0x3000, 0x4000, 4, 4, 4, 4, 12, 0), b"12 bits"),
        (N.WarpPair(0x1000, 0x2000, 0x3004, 0x4000, 4, 4, 4, 4, 8, 0), b"aligned"),
        (N.WarpPair(0x1001, 0x2000, 0x3000, 0x4000, 4, 4, 4, 4, 16, 0), b"aligned"),
    ]
    for bad, msg in cases:
        assert lib.b200_warp_error_workspace_bytes(table(good, bad), 2) == -1
        assert msg in lib.b200_last_error() and b"pair 1" in lib.b200_last_error()
    assert lib.b200_warp_error_workspace_bytes(table(good), 0) == -1 and b"1 to 32" in lib.b200_last_error()
    assert lib.b200_warp_error_workspace_bytes(table(*[good] * 33), 33) == -1
    assert lib.b200_warp_error_workspace_bytes(None, 1) == -1
    sums, ws = C.c_void_p(0x5000), C.c_void_p(0x6000)
    assert lib.b200_warp_error(table(good), 1, sums, None, None, ws, one - 8, None) == 3       # B200_ERR_WORKSPACE
    assert b"need %d bytes" % one in lib.b200_last_error()
    assert lib.b200_warp_error(table(good), 1, None, None, None, ws, one, None) == 1
    assert lib.b200_warp_error(table(good), 1, sums, None, None, C.c_void_p(0x6004), one, None) == 1
