"""Batched RAFT: the batched correlation entry points (b200_corr_*_batch), RAFT.forward on B pairs,
RAFT.forward_sequence and the windowed pre-pass.  Every comparison is bit for bit (torch.equal / file bytes) against
the same work done one pair at a time: the kernels are batch-invariant (a sample's arithmetic does not depend on the
others), so no tolerance is needed."""
import argparse
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from b200 import _native as N
from b200 import nn as K
from nets_common import seeded_weights
from test_aux_kernels_gpu import _lookup_coords

pytestmark = pytest.mark.gpu
DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "all-in-one-deflicker_b200")
GRIDS = [(9, 11), (45, 80), (54, 96), (135, 240)]


def _batch_sizes(H8, W8):
    return (1, 2, 3) if H8 * W8 > 10000 else (1, 2, 3, 7)      # 135 x 240: 5.6 GB per pyramid


def _coords(B, H8, W8, seed):
    """Per-sample coordinates: the all-pairs lookup test's edge cases (outside the map, +-1e3, +-1e7) and a few NaNs."""
    cs = []
    for b in range(B):
        c = _lookup_coords(H8, W8, seed + b)
        c[0, 0, 0, 1] = float("nan")
        c[0, 1, H8 - 1, W8 - 2] = float("nan")
        cs.append(c)
    return torch.cat(cs).to(DEV)


@pytest.mark.parametrize("H8,W8", GRIDS)
def test_batched_builders_and_lookup_equal_single_pairs(H8, W8):
    for B in _batch_sizes(H8, W8):
        g = torch.Generator().manual_seed(B * 100 + H8)
        f1 = torch.randn(B, 256, H8, W8, generator=g).to(DEV)
        f2 = torch.randn(B, 256, H8, W8, generator=g).to(DEV)
        coords = _coords(B, H8, W8, H8 + W8 + B)
        for impl in ("tc", "simt"):
            pyr = K.corr_build_batch(f1, f2, impl=impl)
            assert pyr.shape == (B, N.lib().b200_corr_pyramid_floats(H8, W8))
            for r in range(1, 9):
                got = K.corr_lookup_batch(pyr, coords, r)
                for b in range(B):
                    if r == 1:
                        single = K.corr_build(f1[b:b + 1].contiguous(), f2[b:b + 1].contiguous(), impl=impl)
                        assert torch.equal(pyr[b], single), f"{impl} {H8}x{W8} B={B} sample {b}: pyramid differs"
                        del single
                    want = K.corr_lookup(pyr[b].contiguous(), coords[b:b + 1].contiguous(), r)
                    assert torch.equal(got[b:b + 1].isnan(), want.isnan())
                    assert torch.equal(got[b:b + 1].nan_to_num(), want.nan_to_num()), f"{impl} B={B} r={r} sample {b}"
            del pyr
        torch.cuda.empty_cache()
    print(f"batched corr {H8}x{W8}: both builders and lookup radius 1..8 == single-pair calls (bound: exact)")


@pytest.mark.parametrize("H8,W8", GRIDS)
def test_batched_on_the_fly_correlation_equals_single_pairs(H8, W8):
    for B in (1, 2, 3, 7):
        g = torch.Generator().manual_seed(B * 7 + W8)
        f1 = torch.randn(B, 256, H8, W8, generator=g).to(DEV)
        f2 = torch.randn(B, 256, H8, W8, generator=g).to(DEV)
        coords = _coords(B, H8, W8, 3 * H8 + B)
        state = K.corr_alt_build_batch(f1, f2)
        assert state.shape == (B, N.lib().b200_corr_alt_floats(256, H8, W8))
        singles = [K.corr_alt_build(f1[b:b + 1].contiguous(), f2[b:b + 1].contiguous()) for b in range(B)]
        for b in range(B):
            assert torch.equal(state[b], singles[b])
        for r in range(1, 9):
            got = K.corr_alt_lookup_batch(state, coords, 256, r)
            for b in range(B):
                want = K.corr_alt_lookup(singles[b], coords[b:b + 1].contiguous(), 256, r)
                assert torch.equal(got[b:b + 1].isnan(), want.isnan())
                assert torch.equal(got[b:b + 1].nan_to_num(), want.nan_to_num()), f"B={B} r={r} sample {b}"
    print(f"batched on-the-fly corr {H8}x{W8}: state and lookup radius 1..8 == single-pair calls (bound: exact)")


def test_batched_entry_points_validate_their_arguments():
    f = torch.zeros(2, 256, 9, 11, device=DEV)
    lib = N.lib()
    pyr = K.corr_build_batch(f, f, impl="simt")
    coords = torch.zeros(2, 2, 9, 11, device=DEV)
    out = torch.empty(2, 4 * 81, 9, 11, device=DEV)
    assert lib.b200_corr_lookup_batch(N.ptr(pyr), N.ptr(coords), N.ptr(out), 0, 9, 11, 4, None) != 0
    assert b"batch" in lib.b200_last_error()
    assert lib.b200_corr_lookup_batch(N.ptr(pyr), N.ptr(coords), N.ptr(out), 2, 9, 11, 9, None) != 0
    assert b"radius" in lib.b200_last_error()
    assert lib.b200_corr_build_tc_batch_workspace_bytes(0, 256, 9, 11) == -1
    state = K.corr_alt_build_batch(f, f)
    assert lib.b200_corr_alt_lookup_batch(N.ptr(state), N.ptr(coords), N.ptr(out), 256, 0, 9, 11, 4, None) != 0
    assert b"batch" in lib.b200_last_error()
    assert lib.b200_corr_alt_build_batch(N.ptr(f), N.ptr(f), 2, 100, 9, 11, N.ptr(state), None) != 0
    assert b"dim" in lib.b200_last_error()
    with pytest.raises(N.B200Error, match="another batch"):
        K.corr_lookup_batch(pyr, coords[:1].contiguous())
    with pytest.raises(N.B200Error, match="batch 1"):
        K.corr_build(f, f)


def _raft(golden_dir, mixed=True, alternate=False):
    from src.models.stage_1.core.raft import RAFT
    fx = torch.load(os.path.join(golden_dir, "raft_full.pt"))
    model = RAFT(argparse.Namespace(small=False, mixed_precision=mixed, alternate_corr=alternate))
    model.load_state_dict(seeded_weights(fx["shapes"], fx["seed"]), strict=False)
    return model.to(DEV).eval(), fx


def _three_pairs(fx, seed):
    g = torch.Generator().manual_seed(seed)
    a, b = fx["im1"], fx["im2"]
    noise = (torch.rand(1, 3, 128, 192, generator=g) * 255)
    im1 = torch.cat([a, b, torch.roll(a, (2, -3), (2, 3))])
    im2 = torch.cat([b, noise, a])
    return im1.to(DEV), im2.to(DEV)


def _eager(model):
    class _Ctx:
        def __enter__(self):
            model.args.cuda_graph = False

        def __exit__(self, *exc):
            model.args.cuda_graph = True
    return _Ctx()


@pytest.mark.parametrize("mixed", [True, False])
@pytest.mark.parametrize("alternate", [False, True])
def test_batched_raft_equals_single_pairs(golden_dir, mixed, alternate):
    """A batch of 3 different pairs: every sample equals its own B = 1 forward, in test mode (captured graph, replayed
    twice with new inputs), eagerly with the per-iteration list, and with flow_init."""
    model, fx = _raft(golden_dir, mixed, alternate)
    for seed in (1, 2):                                     # second round: the batch-3 graph replayed on new inputs
        im1, im2 = _three_pairs(fx, seed)
        lo, up = model(im1, im2, iters=3, test_mode=True)
        for b in range(3):
            lo1, up1 = model(im1[b:b + 1], im2[b:b + 1], iters=3, test_mode=True)
            assert torch.equal(lo[b:b + 1], lo1) and torch.equal(up[b:b + 1], up1), f"test mode, round {seed}, sample {b}"
    init = (torch.randn(3, 2, 16, 24, generator=torch.Generator().manual_seed(4)) * 2).to(DEV)
    preds = model(im1, im2, iters=3, flow_init=init)
    assert len(preds) == 3
    with _eager(model):
        lo_e, up_e = model(im1, im2, iters=3, flow_init=init, test_mode=True)
    lo_g, up_g = model(im1, im2, iters=3, flow_init=init, test_mode=True)
    assert torch.equal(lo_e, lo_g) and torch.equal(up_e, up_g)
    for b in range(3):
        one = model(im1[b:b + 1], im2[b:b + 1], iters=3, flow_init=init[b:b + 1].contiguous())
        assert all(torch.equal(p[b:b + 1], q) for p, q in zip(preds, one)), f"iteration list, sample {b}"
        lo1, up1 = model(im1[b:b + 1], im2[b:b + 1], iters=3, flow_init=init[b:b + 1].contiguous(), test_mode=True)
        assert torch.equal(lo_g[b:b + 1], lo1) and torch.equal(up_g[b:b + 1], up1)
    print(f"RAFT mixed={mixed} alternate_corr={alternate}: batch of 3 == 3 single pairs (bound: exact)")


@pytest.mark.parametrize("alternate", [False, True])
def test_forward_sequence_equals_forward_both(golden_dir, alternate):
    """5 frames: the 4 forward and 4 backward flows equal four forward_both calls; padded to 6 pairs (the tail window
    of a longer video) they are the same bits, and the padded call reuses one graph for a 3-frame window."""
    model, fx = _raft(golden_dir, True, alternate)
    g = torch.Generator().manual_seed(9)
    base = torch.cat([fx["im1"], fx["im2"]])
    frames = torch.cat([base, torch.roll(fx["im2"], (1, 2), (2, 3)), (torch.rand(2, 3, 128, 192, generator=g) * 255)])
    frames = frames.to(DEV)
    (lo_f, up_f), (lo_b, up_b) = model.forward_sequence(frames, iters=3)
    assert up_f.shape == up_b.shape == (4, 2, 128, 192)
    for k in range(4):
        (l12, u12), (l21, u21) = model.forward_both(frames[k:k + 1], frames[k + 1:k + 2], iters=3)
        assert torch.equal(lo_f[k:k + 1], l12) and torch.equal(up_f[k:k + 1], u12), f"forward flow {k}"
        assert torch.equal(lo_b[k:k + 1], l21) and torch.equal(up_b[k:k + 1], u21), f"backward flow {k}"
    (plo_f, pup_f), (plo_b, pup_b) = model.forward_sequence(frames, iters=3, pad_to=6)
    assert torch.equal(pup_f, up_f) and torch.equal(pup_b, up_b) and torch.equal(plo_f, lo_f) and torch.equal(plo_b, lo_b)
    keys = len(model._graph_state)
    (_, tup_f), (_, tup_b) = model.forward_sequence(frames[2:], iters=3, pad_to=6)
    assert len(model._graph_state) == keys, "the padded tail captured a graph of its own"
    assert torch.equal(tup_f, up_f[2:]) and torch.equal(tup_b, up_b[2:])
    print(f"forward_sequence (alternate_corr={alternate}): == forward_both x 4, padded tail included (bound: exact)")


# ---- the windowed pre-pass ----

def _clip(root, T=11, H=360, W=640, seed=3):
    import cv2
    vid = root / "clip"
    vid.mkdir()
    g = np.random.default_rng(seed)
    base = (g.random((H // 8, W // 8, 3)) * 255).astype(np.float32)
    base = cv2.resize(base, (W + 64, H + 64), interpolation=cv2.INTER_CUBIC)
    for t in range(T):
        frame = np.clip(base[2 * t:2 * t + H, 3 * t:3 * t + W] + g.normal(0, 2, (H, W, 3)), 0, 255).astype(np.uint8)
        cv2.imwrite(str(vid / f"{t:05d}.png"), frame)
    return vid


def _per_pair(vid, out_dir):
    """The per-pair pre-pass: one compute_flow_both call and two np.save calls per pair."""
    from src.models.stage_1.raft_wrapper import RAFTWrapper
    torch.manual_seed(0)
    raft = RAFTWrapper(model_path=None, max_long_edge=2000)
    frames = sorted(vid.glob("*.png"))
    out_dir.mkdir()
    for a, b in zip(frames, frames[1:]):
        fwd, bwd = raft.compute_flow_both(*raft.load_images(str(a), str(b)))
        np.save(out_dir / f"{a.name}_{b.name}.npy", fwd)
        np.save(out_dir / f"{b.name}_{a.name}.npy", bwd)


def _run_prepass(vid, rank=0, world=1, max_flows=6):
    """src/preprocess_optical_flow.preprocess in a process of its own (random weights seeded like _per_pair), with
    windows of at most max_flows / 2 pairs so that 10 pairs end in a ragged window."""
    code = (f"import sys, torch, argparse; from pathlib import Path; sys.path.insert(0, {PKG!r}); "
            f"from src import preprocess_optical_flow as pp; pp.MAX_FLOWS_PER_BATCH = {max_flows}; "
            f"torch.manual_seed(0); "
            f"pp.preprocess(argparse.Namespace(vid_path=Path({str(vid)!r}), max_long_edge=2000), {rank}, {world})")
    env = dict(os.environ, PYTHONPATH=PKG, B200_ALLOW_RANDOM_RAFT="1")
    return subprocess.Popen([sys.executable, "-c", code], cwd=str(vid.parent), env=env,
                            stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)


def _wait(*procs):
    for p in procs:
        out, _ = p.communicate(timeout=900)
        assert p.returncode == 0, out[-3000:]


def _files(d):
    return {p.name: p.read_bytes() for p in sorted(Path(d).glob("*.npy"))}


@pytest.fixture(scope="module")
def reference_flows(tmp_path_factory):
    root = tmp_path_factory.mktemp("prepass")
    vid = _clip(root)
    _per_pair(vid, root / "per_pair")
    return vid, _files(root / "per_pair")


def test_windowed_prepass_writes_the_per_pair_files(reference_flows):
    vid, want = reference_flows
    flow_dir = vid.parent / "clip_flow"
    _wait(_run_prepass(vid))
    got = _files(flow_dir)
    assert len(want) == 20 and set(got) == set(want)
    assert all(got[k] == want[k] for k in want), [k for k in want if got[k] != want[k]]
    arr = np.load(flow_dir / "00000.png_00001.png.npy")
    assert arr.shape == (360, 640, 2) and arr.dtype == np.float32
    # a partly computed folder is completed; the files already there keep their bytes and mtimes
    for p in (0, 3, 4, 7):                                                 # both files gone: recomputed
        (flow_dir / f"{p:05d}.png_{p + 1:05d}.png.npy").unlink()
        (flow_dir / f"{p + 1:05d}.png_{p:05d}.png.npy").unlink()
    (flow_dir / "00009.png_00010.png.npy").unlink()                        # pair 9 keeps only its backward file
    keep = {p.name: p.stat().st_mtime_ns for p in flow_dir.glob("*.npy")}
    _wait(_run_prepass(vid))
    got = _files(flow_dir)
    assert not (flow_dir / "00009.png_00010.png.npy").exists(), "a pair with one file present is skipped"
    assert all(got[k] == want[k] for k in got)
    assert all((flow_dir / k).stat().st_mtime_ns == t for k, t in keep.items() if k in got)
    assert set(got) == set(want) - {"00009.png_00010.png.npy"}
    print("windowed pre-pass: 20 files byte-identical to the per-pair path; a partial folder is completed")


def test_windowed_prepass_in_two_processes_sharing_one_gpu(reference_flows):
    vid, want = reference_flows
    flow_dir = vid.parent / "clip_flow"
    for f in flow_dir.glob("*.npy"):
        f.unlink()
    _wait(_run_prepass(vid, 0, 2), _run_prepass(vid, 1, 2))
    got = _files(flow_dir)
    assert set(got) == set(want) and all(got[k] == want[k] for k in want)
    print("windowed pre-pass, 2 ranks on one GPU: the per-pair files byte for byte")
