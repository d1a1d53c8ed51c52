"""Host side of overlapping clips (`--clips --clip_overlap V`), no GPU involved: the plan with an overlap, its seams,
the cross-fade weights, the frames each clip writes, the seam-to-rank assignment, the refusals, the seam pairs of the
flicker measurement and the driver's flag.  tests/test_clip_overlap_gpu.py runs the stitch on the GPU."""
import importlib.util
import os
import runpy
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "all-in-one-deflicker_b200")
if PKG not in sys.path:
    sys.path.insert(0, PKG)

from b200 import _native as N  # noqa: E402
from b200 import atlas as A    # noqa: E402

CASES = [(4, 1), (7, 2), (10, 3), (13, 4), (50, 8), (64, 1), (64, 21), (200, 8), (200, 66)]


def _old_plan(T, M):
    """The plan of contiguous clips as it was before the overlap: K = ceil(T / M) ranges of frame_range."""
    K = max(1, -(-T // M))
    return [A.frame_range(k, K, T) for k in range(K)]


@pytest.mark.parametrize("M,V", CASES)
def test_plan_with_overlap_covers_the_video(M, V):
    for T in range(1, 1001):
        plan = A.clip_plan(T, M, V)
        K = len(plan)
        if T <= M:
            assert plan == [(0, T)]
            continue
        assert K == -(-(T - V) // (M - V)), (T, M, V)
        # K is the least: K - 1 clips of at most M frames sharing V frames cover at most (K - 1) M - (K - 2) V
        assert (K - 1) * M - (K - 2) * V < T
        assert plan[0][0] == 0 and plan[-1][1] == T
        assert all(plan[k][0] < plan[k + 1][0] and plan[k][1] < plan[k + 1][1] for k in range(K - 1))
        assert all(plan[k][1] - plan[k + 1][0] == V for k in range(K - 1))
        lengths = [c1 - c0 for c0, c1 in plan]
        assert max(lengths) <= M and max(lengths) - min(lengths) <= 1
        # the two overlap zones of a clip never meet: each clip keeps at least one frame of its own
        seams = A.clip_seams(plan)
        for k, (c0, c1) in enumerate(plan):
            a, b = A.clip_own_frames((c0, c1), T, V)
            assert a == (seams[k - 1][1] if k > 0 else 0) and b == (seams[k][0] if k < K - 1 else T)
            assert b - a >= 1, (T, M, V, k)
        # every frame is written exactly once: by its clip alone, or by the stitch of one seam
        writers = np.zeros(T, np.int64)
        for clip in plan:
            a, b = A.clip_own_frames(clip, T, V)
            writers[a:b] += 1
        for a, b in seams:
            assert b - a == V
            writers[a:b] += 1
        assert (writers == 1).all(), (T, M, V)


@pytest.mark.parametrize("M", [1, 2, 3, 6, 7, 64, 200])
def test_no_overlap_is_the_contiguous_plan(M):
    for T in range(1, 1001):
        plan = A.clip_plan(T, M, 0)
        assert plan == A.clip_plan(T, M) == _old_plan(T, M)
        assert all(a == b for a, b in A.clip_seams(plan))
        assert all(A.clip_own_frames(c, T, 0) == c for c in plan)


def test_the_fifteen_frame_plan_of_the_gpu_tests():
    plan = A.clip_plan(15, 7, 2)
    assert plan == [(0, 7), (5, 11), (9, 15)]
    assert A.clip_seams(plan) == [(5, 7), (9, 11)]
    assert [A.clip_own_frames(c, 15, 2) for c in plan] == [(0, 5), (7, 9), (11, 15)]
    # the measurement's size: V = 0 and V = 8 both give three clips of a 120-frame video at M = 50
    assert len(A.clip_plan(120, 50, 0)) == len(A.clip_plan(120, 50, 8)) == 3


@pytest.mark.parametrize("M,V", [(1, 1), (3, 1), (6, 2), (7, 3), (200, 67)])
def test_too_large_an_overlap_is_refused(M, V):
    with pytest.raises(N.B200Error, match=rf"clip overlap {V} with maximum_number_of_frames {M}"):
        A.clip_plan(10 * M, M, V)
    with pytest.raises(N.B200Error, match=rf"clip overlap {V}"):
        A.clip_plan(1, M, V)                                     # whatever T is
    A.clip_plan(10 * M, M, (M - 1) // 3)                         # the largest V allowed


def test_negative_overlap_is_refused():
    with pytest.raises(N.B200Error, match=r"clip overlap -1 with maximum_number_of_frames 50"):
        A.clip_plan(120, 50, -1)
    with pytest.raises(N.B200Error, match=r"clip overlap -1"):
        A.video_clips(dict(maximum_number_of_frames=50), 120, -1)


def test_video_clips_passes_the_overlap_and_keeps_the_checkpoint_refusal():
    cfg = dict(maximum_number_of_frames=7, load_checkpoint=False)
    assert A.video_clips(cfg, 15, 2) == [(0, 7), (5, 11), (9, 15)]
    assert A.video_clips(cfg, 15) == A.clip_plan(15, 7)
    with pytest.raises(N.B200Error, match="load_checkpoint resumes one atlas"):
        A.video_clips(dict(cfg, load_checkpoint=True, checkpoint_path="ck"), 15, 2)


def test_weights_ramp_linearly_over_the_overlap():
    assert A.seam_weights(0) == []
    assert A.seam_weights(1) == [0.5]
    assert A.seam_weights(2) == [1 / 3, 2 / 3]
    for V in range(1, 40):
        w = A.seam_weights(V)
        assert w == [(j + 1) / (V + 1) for j in range(V)]
        assert all(0.0 < x < 1.0 for x in w)
        # equal steps from clip k's render (w = 0, the frame before the seam) to clip k+1's (w = 1, the frame after)
        steps = np.diff([0.0] + w + [1.0])
        assert np.allclose(steps, 1.0 / (V + 1), rtol=0, atol=1e-15)


def test_seams_are_spread_over_the_ranks_as_a_disjoint_cover():
    for K in range(1, 20):
        seams = A.clip_seams(A.clip_plan(K * 5 - (K - 1), 5, 1))
        assert len(seams) == K - 1
        for world in range(1, 9):
            owned = [A.rank_seams(seams, r, world) for r in range(world)]
            flat = sorted(k for o in owned for k in o)
            assert flat == list(range(K - 1))
            for r, o in enumerate(owned):
                assert o == [k for k in range(K - 1) if k % world == r]


def _flicker():
    spec = importlib.util.spec_from_file_location("evaluate_flicker", os.path.join(PKG, "src", "evaluate_flicker.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_boundary_pairs_without_and_with_an_overlap():
    script = _flicker()
    plan, pairs = script.clip_boundaries(500)                    # maximum_number_of_frames = 200
    assert script.clip_boundaries(500, 0) == (plan, pairs) == ([(0, 167), (167, 334), (334, 500)], [166, 333])
    plan, pairs = script.clip_boundaries(500, 8)
    assert plan == A.clip_plan(500, 200, 8)
    (a0, b0), (a1, b1) = A.clip_seams(plan)
    # the step into the ramp, the V - 1 steps inside it and the step out: V + 1 pairs per seam
    assert pairs == list(range(a0 - 1, b0)) + list(range(a1 - 1, b1)) and len(pairs) == 2 * 9
    scores = [(3.0 * (10.0 if t in pairs else 1.0), 1.0) for t in range(499)]
    doc = script.report("v", 499, {"final": (4, 4)}, {"final": "x"}, {"final": scores}, (plan, pairs))
    assert doc["clips"]["boundary_pairs"] == pairs
    assert doc["sequences"]["final"]["E_boundary"] == 10.0 and doc["sequences"]["final"]["E_interior"] == 1.0


def test_flicker_refuses_an_overlap_without_clips():
    r = subprocess.run([sys.executable, os.path.join(PKG, "src", "evaluate_flicker.py"), "--video_name", "v",
                        "--clip_overlap", "2"], env=dict(os.environ, PYTHONPATH=PKG), capture_output=True, text=True,
                       timeout=300)
    assert r.returncode != 0 and "--clip_overlap is only meaningful with --clips" in r.stderr


@pytest.mark.parametrize("script", ["stage1_neural_atlas.py", "stage1_neural_atlas_seg.py"])
def test_stage1_refuses_an_overlap_without_clips(script, tmp_path):
    r = subprocess.run([sys.executable, os.path.join(PKG, "src", script), "--vid_name", "v", "--clip_overlap", "2"],
                       cwd=str(tmp_path), env=dict(os.environ, PYTHONPATH=PKG), capture_output=True, text=True,
                       timeout=300)
    assert r.returncode != 0 and "--clip_overlap is only meaningful with --clips" in r.stderr
    assert not os.path.exists(str(tmp_path / "results"))


@pytest.mark.parametrize("script", ["stage1_neural_atlas.py", "stage1_neural_atlas_seg.py"])
def test_stage1_refuses_too_large_an_overlap_before_any_work(script, tmp_path):
    import cv2
    os.makedirs(str(tmp_path / "data" / "test" / "v"))
    for t in range(300):
        cv2.imwrite(str(tmp_path / "data" / "test" / "v" / ("%05d.png" % t)), np.zeros((8, 8, 3), np.uint8))
    r = subprocess.run([sys.executable, os.path.join(PKG, "src", script), "--vid_name", "v", "--clips",
                        "--clip_overlap", "67"], cwd=str(tmp_path), env=dict(os.environ, PYTHONPATH=PKG),
                       capture_output=True, text=True, timeout=300)
    assert r.returncode != 0 and "clip overlap 67 with maximum_number_of_frames 200" in r.stderr
    assert not os.path.exists(str(tmp_path / "data" / "test" / "v_flow"))


def test_driver_forwards_the_overlap_to_stage1_and_flicker_only(tmp_path, monkeypatch):
    import cv2
    os.makedirs(str(tmp_path / "data" / "test" / "long"))
    for t in range(3):
        cv2.imwrite(str(tmp_path / "data" / "test" / "long" / ("%05d.png" % t)), np.zeros((8, 8, 3), np.uint8))
    monkeypatch.chdir(tmp_path)
    calls = []
    monkeypatch.setattr(subprocess, "call", lambda cmd, *a, **k: calls.append(list(cmd)) or 0)
    for extra in (["--clips"], ["--clips", "--clip_overlap", "0"], ["--clips", "--clip_overlap", "3"],
                  ["--clips", "--clip_overlap", "3", "--gpus", "2"]):
        calls.clear()
        monkeypatch.setattr(sys, "argv", ["test.py", "--video_frame_folder", "long", "--evaluate_flicker"] + extra)
        with pytest.raises(SystemExit) as e:
            runpy.run_path(os.path.join(PKG, "test.py"), run_name="__main__")
        assert e.value.code == 0
        stage1, stage2, flicker = calls
        assert flicker[1].endswith("evaluate_flicker.py")
        forwarded = "3" in extra
        for cmd in (stage1, flicker):
            assert ("--clip_overlap" in cmd) == forwarded
            if forwarded:
                assert cmd[cmd.index("--clip_overlap") + 1] == "3"
        assert "--clip_overlap" not in stage2
        if not forwarded:            # today's command lines
            assert stage1[-1] == "--clips" and flicker[-1] == "--clips"
    for bad in (["--clip_overlap", "2"], ["--clips", "--clip_overlap", "-1"]):
        monkeypatch.setattr(sys, "argv", ["test.py", "--video_frame_folder", "long"] + bad)
        calls.clear()
        with pytest.raises(SystemExit) as e:
            runpy.run_path(os.path.join(PKG, "test.py"), run_name="__main__")
        assert e.value.code != 0 and calls == []
