"""Host side of fitting a long video as clips (`--clips`), no GPU involved: the clip plan, the clips each rank fits,
the driver's flag and the two refusals."""
import json
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


def _frames(folder, n):
    import cv2
    os.makedirs(folder, exist_ok=True)
    for t in range(n):
        cv2.imwrite(os.path.join(folder, "%05d.png" % t), np.full((16, 24, 3), 10 * t, np.uint8))


def _config(work, **kw):
    cfg = json.load(open(os.path.join(PKG, "src", "config", "config_flow_100.json")))
    cfg.update(kw)
    path = str(work / "cfg.json")
    json.dump(cfg, open(path, "w"))
    return cfg, path


@pytest.mark.parametrize("M", [1, 2, 3, 6, 7, 64, 200])
def test_clip_plan_covers_the_video_in_order(M):
    for T in range(1, 1001):
        clips = A.clip_plan(T, M)
        K = -(-T // M)
        assert len(clips) == K, (T, M)
        assert clips[0][0] == 0 and clips[-1][1] == T
        assert all(clips[i][1] == clips[i + 1][0] for i in range(K - 1))
        lengths = [c1 - c0 for c0, c1 in clips]
        assert max(lengths) <= M and min(lengths) >= 1
        assert max(lengths) - min(lengths) <= 1
        if T <= M:
            assert clips == [(0, T)]
        if M >= 6 and K > 1:
            assert min(lengths) >= 3          # every clip has at least two flow pairs


def test_rank_clips_are_a_disjoint_cover():
    for K in range(1, 20):
        clips = A.clip_plan(K * 6, 6)
        for world in range(1, 9):
            owned = [A.rank_clips(clips, r, world) for r in range(world)]
            flat = [c for o in owned for c in o]
            assert sorted(flat) == clips and len(flat) == len(set(flat))
            for r, o in enumerate(owned):
                assert o == [clips[k] for k in range(K) if k % world == r]


def test_clip_folder_names():
    assert A.clip_name((0, 5)) == "clip_00000_00005"
    assert A.clip_name((195, 13000)) == "clip_00195_13000"


def test_driver_passes_clips_to_stage1_only(tmp_path, monkeypatch):
    _frames(str(tmp_path / "data" / "test" / "long"), 3)
    monkeypatch.chdir(tmp_path)
    calls = []
    monkeypatch.setattr(subprocess, "call", lambda cmd, *a, **k: calls.append(list(cmd)) or 0)
    for extra, gpus in (([], 1), (["--clips"], 1), (["--clips", "--gpus", "2"], 2)):
        calls.clear()
        monkeypatch.setattr(sys, "argv", ["test.py", "--video_frame_folder", "long"] + extra)
        with pytest.raises(SystemExit) as e:
            runpy.run_path(os.path.join(PKG, "test.py"), run_name="__main__")
        assert e.value.code == 0
        stage1, stage2 = calls
        assert stage1[1].endswith("stage1_neural_atlas.py") and stage2[1].endswith("neural_filter_and_refinement.py")
        assert ("--clips" in stage1) == ("--clips" in extra)
        assert "--clips" not in stage2
        assert ("--gpus" in stage1) == ("--gpus" in stage2) == (gpus > 1)


def test_checkpoint_with_several_clips_is_refused(tmp_path):
    cfg = dict(maximum_number_of_frames=6, load_checkpoint=True, checkpoint_path="ck/checkpoint")
    assert A.video_clips(cfg, 6) == [(0, 6)]                       # one clip: the checkpoint resumes it
    with pytest.raises(N.B200Error, match="load_checkpoint resumes one atlas"):
        A.video_clips(cfg, 13)
    assert len(A.video_clips(dict(cfg, load_checkpoint=False), 13)) == 3
    # the script refuses before any work: no flow pre-pass, no GPU
    _frames(str(tmp_path / "data" / "test" / "long"), 13)
    _, path = _config(tmp_path, maximum_number_of_frames=6, load_checkpoint=True)
    env = dict(os.environ, PYTHONPATH=PKG)
    r = subprocess.run([sys.executable, os.path.join(PKG, "src", "stage1_neural_atlas.py"), "--vid_name", "long", "--root",
                        "data/test/", "--config", path, "--clips"], cwd=str(tmp_path), env=env, capture_output=True,
                       text=True, timeout=300)
    assert r.returncode != 0 and "load_checkpoint resumes one atlas" in r.stderr
    assert not os.path.exists(str(tmp_path / "data" / "test" / "long_flow"))


def test_missing_mattes_are_refused_naming_the_clip(tmp_path):
    from src.models.stage_1.unwrap_utils import mask_files
    from src.stage1_neural_atlas_seg import check_clip_mattes
    root = tmp_path / "data" / "test"
    _frames(str(root / "long"), 13)
    _frames(str(root / "long_seg"), 11)                            # the last clip, frames 9..12, lacks two
    clips = A.clip_plan(13, 6)
    assert [len(mask_files(root, "long", c1 - c0, (c0, c1))) for c0, c1 in clips[:2]] == [5, 4]
    with pytest.raises(FileNotFoundError, match=r"11 mask images for clip_00009_00013 \(frames 9 to 12\)"):
        check_clip_mattes(str(root / "long"), clips)
    with pytest.raises(FileNotFoundError, match="11 mask images for 13 frames"):
        mask_files(root, "long", 13)
