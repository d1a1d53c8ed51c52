"""Host-side plan of the windowed RAFT pre-pass (src/preprocess_optical_flow.py): which frames each window decodes,
which pairs it writes, rank blocks, the ragged tail, the skip rule, and the window length chosen from the feature-grid
size and the free device memory.  No GPU."""
import os
import sys

import pytest

from csrc_build import ensure_built

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "all-in-one-deflicker_b200"))

GB = 2 ** 30
H100 = 80 * GB
GRIDS = {"640x360": (45, 80), "1080p": (135, 240), "4K": (270, 480)}


@pytest.fixture(scope="module", autouse=True)
def _built():
    ensure_built()


def _pp():
    from src import preprocess_optical_flow as pp
    return pp


def test_window_plan_covers_the_pairs_in_order():
    pp = _pp()
    # 11 frames, 10 pairs, windows of 4: the tail window is ragged; window [a, b) decodes frames a..b, writes a..b-1
    assert pp.window_plan(list(range(10)), 4) == [(0, 4), (4, 8), (8, 10)]
    assert pp.window_plan(list(range(10)), 1) == [(p, p + 1) for p in range(10)]
    assert pp.window_plan(list(range(10)), 16) == [(0, 10)]
    assert pp.window_plan([], 3) == []
    for k in (1, 2, 3, 5, 8):
        todo = [0, 1, 2, 4, 5, 6, 7, 8, 11]
        wins = pp.window_plan(todo, k)
        assert [p for a, b in wins for p in range(a, b)] == todo          # every pair once, in order
        assert all(1 <= b - a <= k for a, b in wins)


def test_window_plan_never_joins_across_a_skipped_pair():
    pp = _pp()
    # pairs 3 and 9 exist already: no window decodes through them, so 0..2, 4..8 and 10 are runs of their own
    todo = [0, 1, 2, 4, 5, 6, 7, 8, 10]
    assert pp.window_plan(todo, 3) == [(0, 3), (4, 7), (7, 9), (10, 11)]
    frames = [list(range(a, b + 1)) for a, b in pp.window_plan(todo, 3)]
    assert frames == [[0, 1, 2, 3], [4, 5, 6, 7], [7, 8, 9], [10, 11]]


def test_windows_lie_inside_rank_blocks():
    pp = _pp()
    from b200.launch import pair_block
    for T in (11, 80, 7):
        for world in (1, 2, 3, 8):
            seen = []
            for rank in range(world):
                p0, p1 = pair_block(rank, world, T)
                for a, b in pp.window_plan(list(range(p0, p1)), 3):
                    assert p0 <= a < b <= p1
                    seen += list(range(a, b))
            assert seen == list(range(T - 1))


def test_skip_rule_either_file_present(tmp_path):
    pp = _pp()
    vid = tmp_path / "v"
    vid.mkdir()
    frames = [vid / f"{i:05d}.png" for i in range(6)]
    flow_dir = tmp_path / "v_flow"
    flow_dir.mkdir()
    fwd1, _ = pp.flow_files(flow_dir, frames, 1)
    _, bwd3 = pp.flow_files(flow_dir, frames, 3)
    assert fwd1.name == "00001.png_00002.png.npy" and bwd3.name == "00004.png_00003.png.npy"
    fwd1.write_bytes(b"x")
    bwd3.write_bytes(b"x")
    assert pp.pending_pairs(flow_dir, frames, 0, 5) == [0, 2, 4]
    assert pp.pending_pairs(flow_dir, frames, 2, 4) == [2]
    for p in (0, 2, 4):
        for f in pp.flow_files(flow_dir, frames, p):
            f.write_bytes(b"x")
    assert pp.pending_pairs(flow_dir, frames, 0, 5) == []                  # nothing to decode or compute


@pytest.mark.parametrize("size", list(GRIDS))
def test_window_length_from_grid_and_free_memory(size):
    """At least one pair, at most MAX_FLOWS_PER_BATCH / 2 and the pairs left, never decreasing with free memory, and
    when more than one pair is chosen the estimate fits in MEMORY_SHARE of the free memory."""
    pp = _pp()
    from b200 import _native as N
    H8, W8 = GRIDS[size]
    alt = int(N.lib().b200_corr_pyramid_floats(H8, W8)) * 4 > H100 // 2
    floats = N.lib().b200_corr_alt_floats(256, H8, W8) if alt else N.lib().b200_corr_pyramid_floats(H8, W8)
    pixels = 64 * H8 * W8
    frame = pp.ENCODER_BYTES_PER_PIXEL * pixels
    per_flow = 4 * floats + pp.REFINE_BYTES_PER_PIXEL * pixels
    prev = 0
    for free_gb in (0.25, 1, 4, 10, 20, 40, 60, 79):
        k = pp.window_pairs(H8, W8, 1000, free_gb * GB, H100)
        assert 1 <= k <= pp.MAX_FLOWS_PER_BATCH // 2 and k >= prev
        if k > 1:
            assert (k + 1) * frame + 2 * k * per_flow <= pp.MEMORY_SHARE * free_gb * GB
        prev = k
        for left in (1, 2, 5):
            assert pp.window_pairs(H8, W8, left, free_gb * GB, H100) == min(k, left)
    assert pp.window_pairs(H8, W8, 1000, 0, H100) == 1                      # never less than one pair


def test_window_length_on_an_idle_h100():
    """The lengths DESIGN §4b states for an idle 80 GB card (79 GB free): 8 pairs at 640x360 (the cap), 3 at 1080p
    (5.6 GB pyramid per flow), 5 at 4K (on-the-fly correlation: the all-pairs pyramid would take 89 GB)."""
    pp = _pp()
    got = {s: pp.window_pairs(*GRIDS[s], 1000, 79 * GB, H100) for s in GRIDS}
    assert got == {"640x360": 8, "1080p": 3, "4K": 5}
    assert pp.window_pairs(*GRIDS["1080p"], 1000, 79 * GB, H100, alternate_corr=True) == 8
