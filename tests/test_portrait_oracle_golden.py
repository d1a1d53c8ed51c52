"""Both stage-1 oracles and the input producer replayed against the PORTRAIT fixtures (H = 40 > W = 26) frozen from the
reference's own modules by tests/golden/make_golden_portrait.py, and the fixtures' negative controls (one
normalisation swapped for the other) shown to lie far outside the bounds tests/test_portrait_gpu.py applies.  CPU
only."""
import importlib.util
import os
from pathlib import Path

import numpy as np
import pytest
import torch
from PIL import Image

from oracle import atlas_oracle as O
from oracle import seg_oracle as S
from seg_common import ORDER

SPECS = (S.MAPPING1_SPEC, S.MAPPING2_SPEC, S.ATLAS_SPEC, S.ALPHA_SPEC)       # in ORDER
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ("flows_mask", "frames", "flows_rev_mask", "mask_frames", "dx", "dy", "flows_rev", "flows")
MARGIN = 100.0
# the bounds of tests/test_portrait_gpu.py (those of test_atlas_gpu, test_tc_gpu and test_seg_gpu)
LOSS_RTOL_TC = 2e-3          # the loosest loss bound: segmentation variant on the tensor cores
GRAD_FP32 = 1e-3             # max|err| <= 1e-3 max|g| + 2e-4 max|g| of the network, per tensor
ATLAS_GRAD_TC_FRO = 3e-3     # ||err||_F <= 3e-3 ||g||_F per tensor
RENDER_ATOL = 5e-5           # fp32 image, tensor cores
EVAL_UV_ATOL = 2e-6
EVAL_RTOL = 2e-3             # rigidity / flow error: 2e-3 |ref| + a floor (the stored controls are in this unit)


@pytest.fixture(autouse=True)
def _single_thread():
    n = torch.get_num_threads()
    torch.set_num_threads(1)      # fixtures were frozen with 1 thread (addmm summation order)
    yield
    torch.set_num_threads(n)


def picks(n):
    """Indices of the stored entries of a flat gradient (make_golden_portrait.picks)."""
    rest = np.linspace(32, n - 1, 32).round().astype(np.int64) if n > 32 else np.zeros(0, np.int64)
    return np.concatenate([np.arange(min(n, 32)), rest])


def atlas_fixture(golden_dir):
    z = np.load(os.path.join(golden_dir, "portrait.npz"))
    p = np.load(os.path.join(golden_dir, "params_seed1234.npz"))
    mp = [torch.from_numpy(p[f"map{i}"]) for i in range(12)]
    ap = [torch.from_numpy(p[f"atl{i}"]) for i in range(16)]
    data = {k[6:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("video_")}
    return z, data, mp, ap


def seg_fixture(golden_dir):
    z = np.load(os.path.join(golden_dir, "seg_portrait.npz"))
    video = O.Video(**{k[6:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("video_")})
    torch.manual_seed(int(z["init_seed"]))
    nets = S.init_nets()
    for k in ORDER:
        assert float(sum(p.double().sum() for p in nets[k])) == float(z[f"init_{k}_sum"])
    return z, video, torch.from_numpy(z["masks"]), nets


def assert_picks_equal(z, tag, grads):
    for i, g in enumerate(grads):
        gf = g.flatten()
        assert np.array_equal(gf[torch.from_numpy(picks(gf.numel()))].numpy(), z[f"{tag}grad{i}_pick"]), (tag, i)
        assert float(gf.abs().max()) == float(z[f"{tag}grad_max"][i]), (tag, i)


# ------------------------------------------------------------------------------------------------ replay, bit for bit
def test_portrait_geometry(golden_dir):
    z, data, _, _ = atlas_fixture(golden_dir)
    H, W, T = int(z["H"]), int(z["W"]), int(z["T"])
    assert data["frames"].shape == (H, W, 3, T) and H > W
    assert O._half(W) != O._half(max(H, W))


@pytest.mark.parametrize("B", [64, 129])
@pytest.mark.parametrize("it", [0, 6000])
def test_atlas_iteration_bit_exact(golden_dir, B, it):
    z, data, mp, ap = atlas_fixture(golden_dir)
    mp = [p.clone().requires_grad_(True) for p in mp]
    ap = [p.clone().requires_grad_(True) for p in ap]
    terms = O.iteration_losses(O.Video(**data), mp, ap, torch.from_numpy(z[f"inds{B}"]), it)
    terms["total"].backward()
    tag = f"B{B}_it{it}_"
    assert set(terms) == {k[len(tag) + 5:] for k in z.files if k.startswith(tag + "loss_")}
    for k, v in terms.items():
        assert np.float32(v.detach()) == z[tag + "loss_" + k], k
    assert_picks_equal(z, tag, [p.grad for p in mp + ap])


def test_atlas_pretrain_render_eval_bit_exact(golden_dir):
    z, data, mp, ap = atlas_fixture(golden_dir)
    H, W, T = int(z["H"]), int(z["W"]), int(z["T"])
    m = [p.clone().requires_grad_(True) for p in mp]
    opt = torch.optim.Adam(m, lr=1e-4)
    torch.manual_seed(5)
    for f in range(int(z["pre_T"])):
        ys, xs = torch.randint(H, (10000, 1)), torch.randint(W, (10000, 1))
        if f == 0:
            assert np.array_equal(ys.numpy(), z["pre_ys"]) and np.array_equal(xs.numpy(), z["pre_xs"])
        loss = O.pretrain_losses(m, f, ys, xs, int(z["pre_T"]), max(H, W), 0.8)
        opt.zero_grad(); loss.backward()
        if f == 0:
            assert_picks_equal(z, "pre_", [p.grad for p in m])
        opt.step()
        assert np.float32(loss.detach()) == z["pre_losses"][f]
    assert np.array_equal(m[0].detach().flatten()[:64].numpy(), z["pre_w0_head"])
    img = O.render_frame(mp, ap, int(z["render_frame"]), H, W, T)
    assert np.array_equal(img.numpy(), z["render_img"]) and np.array_equal(O.to_uint8(img), z["render_u8"])
    for f in z["eval_frames"]:
        uv, rig, flow = O.eval_maps(O.Video(**data), mp, int(f))
        assert np.array_equal(uv.numpy(), z[f"eval_f{f}_uv"]) and np.array_equal(rig.numpy(), z[f"eval_f{f}_rig"])
        assert np.array_equal(flow.numpy(), z[f"eval_f{f}_flow"])
    assert float(np.abs(z[f"eval_f{T - 1}_flow"]).max()) == 0.0


@pytest.mark.parametrize("it", [0, 6000, 10001])
def test_seg_iteration_bit_exact(golden_dir, it):
    z, video, masks, nets = seg_fixture(golden_dir)
    mine = {k: [p.clone().requires_grad_(True) for p in nets[k]] for k in ORDER}
    terms = S.seg_iteration_losses(video, masks, mine, torch.from_numpy(z["inds"]), it)
    terms["total"].backward()
    tag = f"it{it}_"
    for k, v in terms.items():
        assert np.float32(v.detach()) == z[tag + "loss_" + k], k
    assert_picks_equal(z, tag, [p.grad for k in ORDER for p in mine[k]])


def test_seg_pretrain_and_render_bit_exact(golden_dir):
    z, video, _, nets = seg_fixture(golden_dir)
    H, W, T = video.H, video.W, video.T
    m = [p.clone().requires_grad_(True) for p in nets["mapping1"]]
    opt = torch.optim.Adam(m, lr=1e-4)
    torch.manual_seed(5)
    for f in range(int(z["pre_T"])):
        ys, xs = torch.randint(H, (10000, 1)), torch.randint(W, (10000, 1))
        loss = O.pretrain_losses(m, f, ys, xs, int(z["pre_T"]), max(H, W), 0.8)
        opt.zero_grad(); loss.backward(); opt.step()
        assert np.float32(loss.detach()) == z["pre_losses"][f]
    assert np.array_equal(m[0].detach().flatten()[:64].numpy(), z["pre_w0_head"])
    img, alpha = S.render_frame_seg(nets, int(z["render_frame"]), H, W, T)
    assert np.array_equal(img.numpy(), z["render_img"]) and np.array_equal(alpha.numpy(), z["render_alpha"])
    assert np.array_equal(O.to_uint8(img), z["render_u8"])


def _loader():
    path = os.path.join(ROOT, "all-in-one-deflicker_b200", "src", "models", "stage_1", "unwrap_utils.py")
    spec = importlib.util.spec_from_file_location("our_unwrap_utils", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def write_loader_inputs(tmp, z):
    """The fixture's frames, flows and mattes as the files the loaders read; returns (folder, T)."""
    folder, flow_dir, seg = Path(tmp) / "vid", Path(tmp) / "vid_flow", Path(tmp) / "vid_seg"
    for d in (folder, flow_dir, seg):
        d.mkdir()
    T = sum(1 for k in z.files if k.startswith("frame"))
    names = ["%05d.png" % i for i in range(T)]
    for i in range(T):
        Image.fromarray(z[f"frame{i}"]).save(str(folder / names[i]))
        Image.fromarray(z[f"matte{i}"]).save(str(seg / names[i]))
    for i in range(T - 1):
        np.save(flow_dir / f"{names[i]}_{names[i + 1]}.npy", z[f"f12_{i}"])
        np.save(flow_dir / f"{names[i + 1]}_{names[i]}.npy", z[f"f21_{i}"])
    return folder, T


def test_loaders_bit_exact(golden_dir, tmp_path):
    z = np.load(os.path.join(golden_dir, "loader_portrait.npz"))
    folder, T = write_loader_inputs(tmp_path, z)
    resy, resx = int(z["resy"]), int(z["resx"])
    assert resy > resx and z["f12_0"].shape[:2] == (52, 36)
    assert resy / z["f12_0"].shape[0] != resx / z["f12_0"].shape[1]      # resize_flow's factors differ
    mod = _loader()
    single = mod.load_input_data_single(resy, resx, 200, folder, True, True, folder.parent, "vid")
    seg = mod.load_input_data(resy, resx, 200, folder, True, True, folder.parent, "vid")
    for name, a, b in zip(NAMES, single, seg):
        assert a.shape[:2] == (resy, resx), name
        assert torch.equal(a, torch.from_numpy(z["want_" + name])), name
        want = z["want_seg_mask_frames"] if name == "mask_frames" else z["want_" + name]
        assert torch.equal(b, torch.from_numpy(want)), name + " (load_input_data)"
    assert 0.05 < float(single[0].mean()) < 0.95 and len(np.unique(seg[3].numpy())) > 8


# ------------------------------------------------------------------------------------------------ negative controls
@pytest.mark.parametrize("variant", ["atlas", "seg"])
def test_trip_controls_are_far_outside_the_bounds(golden_dir, variant):
    """Two controls of the trip.  'resx_larger': the gradient rows normalised by max(W, H) (what a trainer passing
    max(H, W), or sample_kernel using half_larger for them, computes).  'larger_resx': every use of larger_dim replaced
    by W (base, rigidity and flow rows and the loss scales), a compound of the loss-head defect and the sampling
    ones; the loss-head scale alone is pinned by test_stage1_heads_gpu's head checks, which are given max(W, H).
    Each control changes a loss term by more than 100 x the loosest loss bound of the GPU tests (2e-3, tensor cores),
    so the trip comparison fails on the losses alone in both precisions.  The gradients move by more than 50 x the
    fp32 gradient bound (1e-3 max|g| plus the per-network floor, which is loose for the small tensors) and more than
    33 x the atlas trip's tensor-core Frobenius bound."""
    z = np.load(os.path.join(golden_dir, "portrait.npz" if variant == "atlas" else "seg_portrait.npz"))
    tags = [f"B{B}_it{it}_" for B in (64, 129) for it in (0, 6000)] if variant == "atlas" else \
        [f"it{it}_" for it in (0, 6000, 10001)]
    for tag in tags:
        for name in ("resx_larger", "larger_resx"):
            key = f"{tag}ctl_{name}"
            assert float(z[key + "_loss"]) >= MARGIN * LOSS_RTOL_TC, (key, float(z[key + "_loss"]))
            dmax, dfro, gm = z[key + "_dmax"], z[key + "_dfro"], z[tag + "grad_max"]
            net = np.repeat(np.arange(4), [2 * s.num_layers for s in SPECS]) if variant == "seg" else \
                np.repeat([0, 1], [12, 16])
            scale = np.array([gm[net == k].max() for k in net])
            assert (dmax / (GRAD_FP32 * gm + 2e-4 * scale)).max() >= MARGIN / 2, key
            if variant == "atlas":
                assert (dfro / (ATLAS_GRAD_TC_FRO * z[tag + "grad_fro"])).max() >= MARGIN / 3, key


def test_pretrain_render_eval_controls_are_far_outside_the_bounds(golden_dir):
    """Pre-training, render and evaluation maps normalised by W where max(W, H) is meant."""
    z = np.load(os.path.join(golden_dir, "portrait.npz"))
    zs = np.load(os.path.join(golden_dir, "seg_portrait.npz"))
    assert float(z["pre_ctl_W_loss"]) >= MARGIN * 1e-4
    gm = z["pre_grad_max"]
    assert (z["pre_ctl_W_dmax"] / (1e-3 * gm)).max() >= MARGIN
    for f in (z, zs):
        assert float(f["render_ctl_W"]) >= MARGIN * RENDER_ATOL
        assert int(f["render_ctl_W_u8"]) >= MARGIN            # the GPU tests require equal u8 images
    for f in z["eval_frames"]:
        assert float(z[f"eval_f{f}_ctl_W_uv"]) >= MARGIN * EVAL_UV_ATOL
    assert float(z["eval_f2_ctl_W_flow"]) >= MARGIN * EVAL_RTOL
    # the rigidity map moves by 47 x and 53 x its bound: the same evaluation's uv map (above) fails by thousands
    for f in z["eval_frames"]:
        assert float(z[f"eval_f{f}_ctl_W_rig"]) >= 20 * EVAL_RTOL
