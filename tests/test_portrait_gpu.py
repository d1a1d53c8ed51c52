"""Both stage-1 variants, pre-training, render, evaluation maps and the input producer on a PORTRAIT video (H = 40 >
W = 26), against the fixtures frozen from the reference by tests/golden/make_golden_portrait.py.  Needs a GPU.

On a landscape video resx == max(resx, resy), so a kernel that normalises the gradient-loss rows by max(W, H), or
anything else by W, passes every landscape test.  Here the halves are 20 and 13.  The bounds are those of
test_atlas_gpu (fp32 trip), test_tc_gpu (tensor-core trip: Frobenius), test_seg_gpu (segmentation trip, render) and
test_stage1_heads_gpu (sampling bit for bit, loss heads within C_ENV of float64 on the device's own outputs);
tests/test_portrait_oracle_golden.py shows every negative control of the fixtures lies far outside them.
"""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import test_stage1_heads_gpu as HD
from b200 import _native as N
from b200 import atlas as A
from b200 import seg as SG
from oracle import atlas_oracle as O
from oracle import seg_oracle as S
from seg_common import ORDER
from test_portrait_oracle_golden import atlas_fixture, picks, seg_fixture, write_loader_inputs

pytestmark = pytest.mark.gpu
DEV = "cuda"
PRECS = [pytest.param(N.PREC_FP32, id="fp32"), pytest.param(N.PREC_TC, id="tc")]


def _need(prec):
    if prec == N.PREC_TC and not N.lib().b200_device_supports_tc():
        pytest.skip("needs sm_90")


def _atlas_trainer(data, mp, ap, B, prec, t0=0, t1=None, resx=None):
    vid = A.DeviceVideo.from_reference_layout(data, DEV, t0, t1)
    tr = A.AtlasTrainer(vid, {"samples_batch": B}, precision=prec, device=DEV, resx=resx)
    tr.load_state(O.state_dict_of(mp), O.state_dict_of(ap))
    return tr


def _seg_trainer(video, masks, nets, B, prec, t0=0, t1=None, resx=None):
    data = dict(frames=video.frames, frames_dx=video.frames_dx, frames_dy=video.frames_dy, flow_fwd=video.flow_fwd,
                flow_bwd=video.flow_bwd, mask_fwd=video.mask_fwd, mask_bwd=video.mask_bwd)
    vid = A.DeviceVideo.from_reference_layout(data, DEV, t0, t1)
    tr = SG.SegTrainer(vid, SG.pack_mask_frames(masks, DEV, t0, t1), {"samples_batch": B}, precision=prec, device=DEV,
                       resx=resx)
    tr.load_state({k: O.state_dict_of(nets[k]) for k in ORDER})
    return tr


def _report(name, worst):
    print(f"portrait {name}: worst error / bound {worst:.3g}")
    assert worst <= 1.0, (name, worst)


# ------------------------------------------------------------------------------------------------ sampling + heads
@pytest.fixture
def portrait_in_heads(golden_dir, monkeypatch):
    """test_stage1_heads_gpu's checks, run on the portrait fixtures instead of the landscape ones."""
    z, data, _, _ = atlas_fixture(golden_dir)
    monkeypatch.setattr(HD, "_golden_video", lambda d: (data, torch.from_numpy(z["inds64"])))
    monkeypatch.setattr(HD, "load_fixture", lambda d: seg_fixture(d))
    return data


ATLAS_CASES = [
    # name, video, B, precision, with_global, pe, masks, world  (test_stage1_heads_gpu.CASES layout)
    ("portrait-fp32-global", "golden", 64, N.PREC_FP32, True, 0, "mixed", 1),
    ("portrait-tc-global", "golden", 64, N.PREC_TC, True, 0, "mixed", 1),
    ("portrait-fp32-local-2shard", "golden", 64, N.PREC_FP32, False, 0, "mixed", 2),
    ("portrait-tc-global-2shard", "golden", 64, N.PREC_TC, True, 0, "mixed", 2),
    ("portrait-B129-fp32-2shard", "golden", 129, N.PREC_FP32, True, 0, "mixed", 2),
    ("portrait-B129-tc", "golden", 129, N.PREC_TC, False, 0, "mixed", 1),
]


@pytest.mark.parametrize("case", ATLAS_CASES, ids=[c[0] for c in ATLAS_CASES])
def test_atlas_sampling_and_head(golden_dir, portrait_in_heads, case):
    H, W = portrait_in_heads["frames"].shape[:2]
    tr = HD._atlas_trainer(portrait_in_heads, golden_dir, 64, N.PREC_FP32, 0)
    assert tr._config(True).resx == W != max(H, W)           # the trainer passes the width, not the larger side
    HD.test_atlas_sampling_and_loss_head(golden_dir, case)


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("world", [1, 2])
def test_seg_sampling_and_head(golden_dir, portrait_in_heads, prec, world):
    _need(prec)
    z, video, masks, nets = seg_fixture(golden_dir)
    assert _seg_trainer(video, masks, nets, 64, prec)._config(0).resx == video.W
    HD.test_seg_trip_glue_and_head(golden_dir, prec, world)


# ------------------------------------------------------------------------------------------------ trips vs fixture
def _net_scale(z, tag, sizes):
    """Per tensor, the largest max|g| of its network: test_seg_gpu's floor for near-cancelling bias gradients (the
    mapping network's two-entry output bias sums every row's gradient; its fp32 atomics reach 1e-3 of its own max)."""
    gm = z[tag + "grad_max"]
    net = np.repeat(np.arange(len(sizes)), sizes)
    return np.array([gm[net == k].max() for k in net])


def _grad_pick_ratio(z, tag, grads, rel, floor=None):
    r = []
    for i, g in enumerate(grads):
        gf = g.flatten().cpu()
        bound = rel * float(z[f"{tag}grad_max"][i]) + (0.0 if floor is None else floor[i]) + 1e-9
        r.append(float((gf[torch.from_numpy(picks(gf.numel()))] - torch.from_numpy(z[f"{tag}grad{i}_pick"]))
                       .abs().max()) / bound)
    print(f"{tag} gradient picks, error / bound per tensor:", " ".join(f"{x:.2f}" for x in r))
    return max(r)


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("B", [64, 129])
@pytest.mark.parametrize("it", [0, 6000])
def test_atlas_trip_matches_fixture(golden_dir, prec, B, it):
    _need(prec)
    z, data, mp, ap = atlas_fixture(golden_dir)
    inds = torch.from_numpy(z[f"inds{B}"])
    tr = _atlas_trainer(data, mp, ap, B, prec)
    tr.indices.copy_(inds.reshape(-1))
    tr.loss_grad(tr.uses_global(it))
    torch.cuda.synchronize()
    tag = f"B{B}_it{it}_"
    keys = ("total", "rgb", "gradient", "rigidity", "rigidity_global", "flow")
    want = [float(z[tag + "loss_" + k]) if tag + "loss_" + k in z.files else 0.0 for k in keys]
    losses = tr.losses.cpu().numpy()[:6]
    rtol = 2e-3 if prec == N.PREC_TC else 2e-4
    worst = max(abs(g - w) / (rtol * abs(w)) for g, w in zip(losses, want) if w != 0)
    assert all(g == 0 for g, w in zip(losses, want) if w == 0)
    grads = [v for which in ("mapping", "atlas") for v in tr.grad_views(which).values()]
    # whole tensors against the oracle's gradients, which equal the fixture's stored entries bit for bit
    # (test_portrait_oracle_golden); fp32: test_atlas_gpu's bound with test_seg_gpu's per-network floor (_net_scale),
    # tensor cores: test_tc_gpu's whole-tensor bound
    m = [p.clone().requires_grad_(True) for p in mp]
    a = [p.clone().requires_grad_(True) for p in ap]
    O.iteration_losses(O.Video(**data), m, a, inds, it)["total"].backward()
    scale = _net_scale(z, tag, (12, 16))
    for i, (g, p) in enumerate(zip(grads, m + a)):
        assert np.array_equal(p.grad.flatten()[torch.from_numpy(picks(p.grad.numel()))].numpy(), z[f"{tag}grad{i}_pick"])
        err = g.cpu() - p.grad
        if prec == N.PREC_FP32:
            worst = max(worst, float(err.abs().max()) / (1e-3 * float(p.grad.abs().max()) + 2e-4 * scale[i]))
        else:
            worst = max(worst, float(err.norm() / (3e-3 * p.grad.norm())))
    _report(f"atlas trip B={B} it={it} {'tc' if prec else 'fp32'}", worst)


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("it", [0, 6000, 10001])
def test_seg_trip_matches_fixture(golden_dir, prec, it):
    _need(prec)
    z, video, masks, nets = seg_fixture(golden_dir)
    tr = _seg_trainer(video, masks, nets, 64, prec)
    tr.indices.copy_(torch.from_numpy(z["inds"]).reshape(-1))
    tr.loss_grad(it)
    torch.cuda.synchronize()
    got = tr.loss_dict()
    tc = prec == N.PREC_TC
    tag = f"it{it}_"
    rtol = 2e-3 if tc else 2e-4
    worst = max(abs(got[k[len(tag) + 5:]] - float(z[k])) / (rtol * abs(float(z[k])))
                for k in z.files if k.startswith(tag + "loss_") and float(z[k]) != 0)
    grads = [g for k in ORDER for g in tr.grad_views(k).values()]
    scale = _net_scale(z, tag, [len(nets[k]) for k in ORDER])
    worst = max(worst, _grad_pick_ratio(z, tag, grads, 1.5e-2 if tc else 1e-3, (2e-3 if tc else 2e-4) * scale))
    _report(f"seg trip it={it} {'tc' if tc else 'fp32'}", worst)


def test_frame_shards_sum_to_the_whole_trip(golden_dir):
    """test_atlas_gpu::test_frame_sharding_is_linear on the portrait video, for both variants."""
    z, data, mp, ap = atlas_fixture(golden_dir)
    inds = torch.from_numpy(z["inds129"]).reshape(-1)
    T = data["frames"].shape[3]
    full = _atlas_trainer(data, mp, ap, 129, N.PREC_FP32)
    full.indices.copy_(inds); full.loss_grad(True)
    acc = torch.zeros_like(full.grad_loss)
    for r in range(2):
        part = _atlas_trainer(data, mp, ap, 129, N.PREC_FP32, *A.frame_range(r, 2, T))
        part.indices.copy_(inds); part.loss_grad(True)
        acc += part.grad_loss
    torch.cuda.synchronize()
    n = full.n_params
    worst = float((acc[:n] - full.grads).abs().max() / (1e-4 * full.grads.abs().max()))
    np.testing.assert_allclose(acc[n:n + 6].cpu().numpy(), full.losses[:6].cpu().numpy(), rtol=1e-5)
    zs, video, masks, nets = seg_fixture(golden_dir)
    sinds = torch.from_numpy(zs["inds"]).reshape(-1)
    full = _seg_trainer(video, masks, nets, 64, N.PREC_FP32)
    full.indices.copy_(sinds); full.loss_grad(0)
    acc = torch.zeros_like(full.grads)
    lacc = torch.zeros_like(full.losses)
    for r in range(2):
        part = _seg_trainer(video, masks, nets, 64, N.PREC_FP32, *A.frame_range(r, 2, video.T))
        part.indices.copy_(sinds); part.loss_grad(0)
        acc += part.grads
        lacc += part.losses
    torch.cuda.synchronize()
    worst = max(worst, float((acc - full.grads).abs().max() / (1e-4 * full.grads.abs().max())))
    np.testing.assert_allclose(lacc[:12].cpu().numpy(), full.losses[:12].cpu().numpy(), rtol=1e-5)
    assert torch.equal(lacc[12:14].cpu(), 2 * full.losses[12:14].cpu())
    _report("frame shards", worst)


# ------------------------------------------------------------------------------------------------ resx = 0
def _same_rows(a, b):
    """Coordinate rows [9][cap][4] of two trips on the same samples: bit for bit, the compacted flow-match groups
    (whose order follows the device's atomics) as sets of rows."""
    keep = [g for g in range(9) if g not in (HD.G_FWD, HD.G_BWD)]
    assert np.array_equal(a[keep].view(np.uint32), b[keep].view(np.uint32)), "resx = 0 does not sample like resx = W"
    for g in (HD.G_FWD, HD.G_BWD):
        assert np.array_equal(HD._sorted_bits(a[g]), HD._sorted_bits(b[g])), f"flow group {g}"


def test_resx_zero_means_the_width_in_both_variants(golden_dir):
    """B200AtlasConfig::resx and B200SegConfig::resx <= 0 stand for the video's width: the sampled coordinate rows are
    bit-identical to resx = W, and the trips agree up to the order of their fp32 atomics."""
    z, data, mp, ap = atlas_fixture(golden_dir)
    H, W = data["frames"].shape[:2]
    inds = torch.from_numpy(z["inds129"])
    out = []
    for resx in (W, 0):
        tr = _atlas_trainer(data, mp, ap, 129, N.PREC_FP32, resx=resx)
        cfg = HD._atlas_cfg(tr, 129, True)
        assert cfg.resx == resx
        v = HD._atlas_views(tr, cfg, HD._atlas_step(tr, cfg, inds, 0))
        out.append((v["x_map"], tr.losses.cpu().numpy().copy(), tr.grads.cpu().clone()))
    _same_rows(out[0][0], out[1][0])
    np.testing.assert_allclose(out[1][1], out[0][1], rtol=1e-5)
    assert float((out[1][2] - out[0][2]).abs().max()) <= 1e-4 * float(out[0][2].abs().max())
    assert np.all(np.isfinite(out[1][1]))
    _, video, masks, nets = seg_fixture(golden_dir)
    sinds = torch.from_numpy(z["inds64"]).reshape(-1).to(DEV)
    seg = []
    for resx in (W, 0):
        tr = _seg_trainer(video, masks, nets, 64, N.PREC_FP32, resx=resx)
        cfg = tr._config(0)
        assert cfg.resx == resx
        ws = torch.zeros(int(tr.lib.b200_seg_workspace_bytes(C.byref(cfg))), dtype=torch.uint8, device=DEV)
        N.check(tr.lib.b200_seg_loss_grad(C.byref(cfg), C.byref(tr.video.struct), N.ptr(tr.mask), N.ptr(sinds),
                                          N.ptr(tr.params), N.ptr(tr.grads), N.ptr(tr.losses), N.ptr(ws), ws.numel(),
                                          N.current_stream()))
        off = (C.c_int64 * N.SEG_OFFSET_FLOATS)()
        N.check(tr.lib.b200_seg_workspace_offsets(C.byref(cfg), N.ptr(ws), off))
        torch.cuda.synchronize()
        xm = ws[off[1]:off[1] + 9 * 128 * 16].view(torch.float32).cpu().numpy().reshape(9, 128, 4)
        seg.append((xm, tr.losses.cpu().numpy().copy(), tr.grads.cpu().clone()))
    _same_rows(seg[0][0], seg[1][0])
    assert np.all(np.isfinite(seg[1][1][:12])) and bool(torch.isfinite(seg[1][2]).all())
    np.testing.assert_allclose(seg[1][1], seg[0][1], rtol=1e-5)
    assert float((seg[1][2] - seg[0][2]).abs().max()) <= 1e-4 * float(seg[0][2].abs().max())


# ------------------------------------------------------------------------------------------------ pre-training
@pytest.mark.parametrize("prec", PRECS)
def test_atlas_pretrain_matches_fixture(golden_dir, prec):
    _need(prec)
    z, data, mp, ap = atlas_fixture(golden_dir)
    H, W = data["frames"].shape[:2]
    Tp, B = int(z["pre_T"]), z["pre_ys"].shape[0]
    tr = _atlas_trainer(data, mp, ap, 64, prec)
    # one b200_pretrain_loss_grad_for on the fixture's rows: coordinates bit for bit, loss and gradient
    cfg = HD._atlas_cfg(tr, B, False)
    ws = torch.full((int(tr.lib.b200_atlas_workspace_bytes_for(C.byref(cfg), C.byref(tr.map_desc))),), 0xFF,
                    dtype=torch.uint8, device=DEV)
    ys = torch.from_numpy(z["pre_ys"].astype(np.int64)).reshape(-1).to(DEV)
    xs = torch.from_numpy(z["pre_xs"].astype(np.int64)).reshape(-1).to(DEV)
    N.check(tr.lib.b200_pretrain_loss_grad_for(C.byref(cfg), C.byref(tr.map_desc), max(H, W), Tp, 0, N.ptr(ys),
                                               N.ptr(xs), N.ptr(tr.params), N.ptr(tr.grads), N.ptr(tr.losses), N.ptr(ws),
                                               ws.numel(), N.current_stream()))
    torch.cuda.synchronize()
    xm = HD._atlas_views(tr, cfg, ws)["x_map"][0, :B]
    hL = np.float32(max(H, W) / 2.0)
    ref = np.stack([HD._norm(z["pre_xs"].reshape(-1).astype(np.float32), hL),
                    HD._norm(z["pre_ys"].reshape(-1).astype(np.float32), hL),
                    np.full(B, np.float32(0 / (Tp / 2.0) - 1.0), np.float32), np.zeros(B, np.float32)], axis=1)
    assert np.array_equal(xm.view(np.uint32), ref.view(np.uint32))
    worst = abs(float(tr.losses[0]) - float(z["pre_losses"][0])) / (1e-4 * float(z["pre_losses"][0]))
    worst = max(worst, _grad_pick_ratio(z, "pre_", list(tr.grad_views("mapping").values()),
                                        1e-3 if prec == N.PREC_FP32 else 1.5e-2))
    # the whole sweep (test_atlas_gpu::test_pretrain_two_steps): same random stream, same rows, Adam on the device
    tr = _atlas_trainer(data, mp, ap, 64, prec)
    torch.manual_seed(5)
    last = tr.pretrain(Tp, H, W, 1)
    torch.cuda.synchronize()
    worst = max(worst, abs(float(last[0]) - float(z["pre_losses"][-1])) / (1e-4 * float(z["pre_losses"][-1])))
    head = tr.param_views("mapping")["hidden.0.weight"].flatten()[:64].cpu().numpy()
    worst = max(worst, float(np.abs(head - z["pre_w0_head"]).max()) / 1e-5)
    _report(f"atlas pretrain {'tc' if prec else 'fp32'}", worst)


@pytest.mark.parametrize("prec", PRECS)
def test_seg_pretrain_matches_fixture(golden_dir, prec):
    """b200_mlp_pretrain_loss_grad through SegTrainer.pretrain, with test_seg_gpu::test_seg_pretrain_matches_oracle's
    bounds (loss rtol 2e-4, weights 5e-5) in fp32 and test_seg_gpu's tensor-core loss bound (rtol 2e-3, weights 2.5e-4,
    the three-step trajectory's) on the tensor cores."""
    _need(prec)
    tc = prec == N.PREC_TC
    z, video, masks, nets = seg_fixture(golden_dir)
    tr = _seg_trainer(video, masks, nets, 64, prec)
    torch.manual_seed(5)
    last = tr.pretrain("mapping1", int(z["pre_T"]), video.H, video.W, 1)
    worst = abs(float(last) - float(z["pre_losses"][-1])) / ((2e-3 if tc else 2e-4) * float(z["pre_losses"][-1]))
    head = tr.param_views("mapping1")["hidden.0.weight"].flatten()[:64].cpu().numpy()
    worst = max(worst, float(np.abs(head - z["pre_w0_head"]).max()) / (2.5e-4 if tc else 5e-5))
    _report(f"seg pretrain {'tc' if tc else 'fp32'}", worst)


# ------------------------------------------------------------------------------------------------ render / evaluation
def _check_u8(u8, ref_img, bound):
    """The u8 frame is the truncation of 255 x the image: equal to the fixture's wherever no value within `bound` of
    the fixture's image truncates differently.  (Under the segmentation variant's tensor-core bound almost every
    value is within reach of an integer: there test_seg_gpu's rule, at most 1 off on under 1 % of the values.)"""
    x = ref_img.astype(np.float64) * 255
    if 255 * bound > 0.05:
        diff = np.abs(u8.astype(int) - x.astype(np.uint8).astype(int))
        assert diff.max() <= 1 and (diff != 0).mean() < 0.01
        return
    decided = np.floor(x - 255 * bound) == np.floor(x + 255 * bound)
    assert decided.mean() > 0.9
    assert np.array_equal(u8[decided], (x[decided]).astype(np.uint8))


@pytest.mark.parametrize("prec", PRECS)
def test_render_matches_fixture(golden_dir, prec):
    """b200_render_for and b200_seg_render in chunks of 300 pixels: the second chunk starts at x = 14 of row 11."""
    _need(prec)
    tc = prec == N.PREC_TC
    z, data, mp, ap = atlas_fixture(golden_dir)
    H, W, _, T = data["frames"].shape
    assert 300 % W != 0
    tr = _atlas_trainer(data, mp, ap, 64, prec)
    img, u8 = tr.render_frame(int(z["render_frame"]), H, W, T, chunk=300, want_u8=True)
    bound = 5e-5 if tc else 2e-5
    worst = float(np.abs(img.cpu().numpy() - z["render_img"]).max()) / bound
    _check_u8(u8.cpu().numpy(), z["render_img"], bound)
    zs, video, masks, nets = seg_fixture(golden_dir)
    st = _seg_trainer(video, masks, nets, 64, prec)
    img, alpha, u8 = st.render_frame(int(zs["render_frame"]), H, W, T, chunk=300, want_u8=True)
    a_bound, i_bound = (2e-3, 5e-3) if tc else (2e-5, 2e-5)
    worst = max(worst, float(np.abs(alpha.cpu().numpy() - zs["render_alpha"]).max()) / a_bound,
                float(np.abs(img.cpu().numpy() - zs["render_img"]).max()) / i_bound)
    _check_u8(u8.cpu().numpy(), zs["render_img"], i_bound)
    _report(f"render {'tc' if tc else 'fp32'}", worst)


@pytest.mark.parametrize("prec", PRECS)
def test_eval_maps_match_fixture(golden_dir, prec):
    """b200_eval_maps of frame 2 and of the last frame, in chunks of 300 pixels (test_atlas_gpu's bounds)."""
    _need(prec)
    z, data, mp, ap = atlas_fixture(golden_dir)
    tr = _atlas_trainer(data, mp, ap, 64, prec)
    T = data["frames"].shape[3]
    worst = 0.0
    for f in (int(v) for v in z["eval_frames"]):
        uv, rig, flow = (x.cpu().numpy() for x in tr.eval_maps(f, chunk=300))
        worst = max(worst, float(np.abs(uv - z[f"eval_f{f}_uv"]).max()) / 2e-6,
                    float((np.abs(rig - z[f"eval_f{f}_rig"]) / (2e-3 * np.abs(z[f"eval_f{f}_rig"]) + 1e-3)).max()),
                    float((np.abs(flow - z[f"eval_f{f}_flow"]) / (2e-3 * np.abs(z[f"eval_f{f}_flow"]) + 2e-4)).max()))
        if f == T - 1:
            assert float(np.abs(flow).max()) == 0.0
        else:
            assert float((flow > 0).mean()) > 0.3
    _report(f"eval maps {'tc' if prec else 'fp32'}", worst)


# ------------------------------------------------------------------------------------------------ input producer
def _reference_pack(z, t0, t1):
    want = {n: torch.from_numpy(z["want_" + n]) for n in ("frames", "dx", "dy", "flows", "flows_rev", "flows_mask",
                                                           "flows_rev_mask")}
    data = dict(frames=want["frames"], frames_dx=want["dx"], frames_dy=want["dy"], flow_fwd=want["flows"],
                flow_bwd=want["flows_rev"], mask_fwd=want["flows_mask"], mask_bwd=want["flows_rev_mask"])
    return A.DeviceVideo.from_reference_layout(data, DEV, t0, t1), want


def test_device_producer_matches_portrait_loader(golden_dir, tmp_path):
    """DeviceVideo.from_files at 44 x 30 from 52 x 36 flows (resize_flow's swapped factors differ from the geometric
    ones): records and bitmaps bit for bit, for the whole video and for the clip of frames [1, 4)."""
    z = np.load(os.path.join(golden_dir, "loader_portrait.npz"))
    folder, T = write_loader_inputs(tmp_path, z)
    resy, resx = int(z["resy"]), int(z["resx"])
    ref, want = _reference_pack(z, 0, T)
    got, frames = A.DeviceVideo.from_files(folder, folder.parent, "vid", resy, resx, 200, DEV)
    torch.cuda.synchronize()
    assert (got.H, got.W, got.T) == (resy, resx, T)
    assert torch.equal(frames, want["frames"])
    n = resy * resx * T * 16
    assert torch.equal(got.records[:n].cpu(), ref.records[:n].cpu())
    words = (resy * resx * T + 31) // 32
    assert torch.equal(got.bits_f[:words].cpu(), ref.bits_f[:words].cpu())
    assert torch.equal(got.bits_b[:words].cpu(), ref.bits_b[:words].cpu())
    # a clip: frames [1, T) of the folder; its first frame has no backward partner inside the clip
    clip, _ = A.DeviceVideo.from_files(folder, folder.parent, "vid", resy, resx, 200, DEV, clip=(1, T))
    torch.cuda.synchronize()
    hw = resy * resx
    rc = clip.records[:hw * (T - 1) * 16].view(T - 1, hw, 16).cpu()
    rr = ref.records[:n].view(T, hw, 16)[1:].cpu()
    assert torch.equal(rc[:, :, :11], rr[:, :, :11]) and torch.equal(rc[:, :, 13], rr[:, :, 13])
    assert torch.equal(rc[1:], rr[1:])
    assert float(rc[0, :, 11:13].abs().max()) == 0.0 and float(rc[0, :, 14].abs().max()) == 0.0


# ------------------------------------------------------------------------------------------------ the atlas script
def test_atlas_script_on_a_portrait_video(tmp_path):
    """stage1_neural_atlas.py on a 6-frame 192 x 128 video: the script fits it at resx = 128 (the width), writes
    192 x 128 frames, and its PSNR marker and frames equal the evaluation of its own checkpoint."""
    import glob
    import json
    import subprocess
    import sys
    import cv2
    from test_pipeline_gpu import PKG, _write_video
    from src.models.stage_1 import driver as D
    from src.models.stage_1 import evaluate as E
    vid, H, W, T, it = "tall", 192, 128, 6, 20
    data = tmp_path / "data" / "test" / vid
    _write_video(str(data), T=T, H=H, W=W)
    assert D.frame_size(str(data), 1) == (W, H)
    cfg = json.load(open(os.path.join(PKG, "src", "config", "config_flow_100.json")))
    cfg.update(iters_num=it + 1, evaluate_every=it, pretrain_iter_number=2, samples_batch=2000, stop_global_rigidity=10)
    json.dump(cfg, open(str(tmp_path / "cfg.json"), "w"))
    env = dict(os.environ, PYTHONPATH=PKG, B200_ALLOW_RANDOM_RAFT="1")     # no pretrained RAFT offline
    for k in ("WORLD_SIZE", "RANK", "LOCAL_RANK"):
        env.pop(k, None)
    r = subprocess.run([sys.executable, os.path.join(PKG, "src", "stage1_neural_atlas.py"), "--vid_name", vid, "--root",
                        "data/test/", "--down", "1", "--config", str(tmp_path / "cfg.json")], cwd=str(tmp_path), env=env,
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    res = tmp_path / "results" / vid / "stage_1"
    outs = sorted(glob.glob(str(res / "output" / "*.png")))
    assert len(outs) == T and all(cv2.imread(o).shape == (H, W, 3) for o in outs)
    marker = glob.glob(str(res / ("%06d" % it) / "PSNR_*"))
    assert len(marker) == 1
    ck = torch.load(str(res / "checkpoint"), weights_only=False)
    video, frames = A.DeviceVideo.from_files(data, data.parent, vid, H, W, cfg["maximum_number_of_frames"], DEV)
    tr = A.AtlasTrainer(video, cfg, precision=D.precision(), device=DEV, resx=W)
    tr.load_checkpoint(ck, optimizer=False)
    out = tmp_path / "eval"
    psnr = E.evaluate_model_single(tr, W, H, T, frames, str(out), it, vid, save_checkpoint=False,
                                   output_folder=str(out / "frames"))
    tr.release()
    assert os.path.basename(marker[0]) == "PSNR_%f" % psnr
    for o in outs:
        with open(o, "rb") as a, open(str(out / "frames" / os.path.basename(o)), "rb") as b:
            assert a.read() == b.read(), o
