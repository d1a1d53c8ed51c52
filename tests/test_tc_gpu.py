"""wgmma path (B200_PREC_TC: 2-term fp16 split, 3 MMAs per product, fp32 accumulation in registers)
against the oracle.  Needs a compute-capability-9 GPU.

Tolerances
  forward       |uv err| <= 5e-6, |atlas output err| <= 5e-5 (PE frequencies up to 2^9*pi amplify the
                uv rounding), against the fp32 oracle
  gradients     measured against a FLOAT64 evaluation of the oracle, per tensor:
                  90th percentile of |err| <= max(10 x the fp32 CUDA-core path's, 2e-3 max|grad|)
                  (the TC forward differs from the fp32 one by ~1e-7 in uv; the 2^9*pi positional frequency
                  turns that into ~1e-5 in rgb and hence ~1e-4 relative in dL/drgb — same mechanism, smaller
                  factor, for the fp32 path against float64)
                  ||err||_F <= 3e-3 ||grad||_F
                ReLU' is discontinuous: any fp32-level implementation flips the mask of the few
                pre-activations that lie within rounding of 0 (~1 per 10^6; each flip changes one row of dW
                by O(1)), so the bulk is compared tightly and the whole tensor in Frobenius norm
"""
import os

import numpy as np
import pytest
import torch

from b200 import _native as N
from b200 import atlas as A
from b200 import synth
from oracle import atlas_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _need_tc():
    if not N.lib().b200_device_supports_tc():
        pytest.skip("no sm_90 device")


def _params(golden_dir):
    z = np.load(os.path.join(golden_dir, "params_seed1234.npz"))
    return ([torch.from_numpy(z[f"map{i}"]) for i in range(12)], [torch.from_numpy(z[f"atl{i}"]) for i in range(16)])


def _tc_outputs(tr, B):
    view = tr.workspace_views()
    cap = view["cap"]
    return cap, view["x_map"].reshape(9 * cap, 4), view["uv"].reshape(9 * cap, 2), view["y_atlas"].reshape(3 * cap, 3)


@pytest.mark.parametrize("B,shape", [(64, (24, 40, 6)), (3000, (60, 100, 9))])
def test_tc_forward_and_gradients(golden_dir, B, shape):
    _need_tc()
    H, W, T = shape
    data = synth.throughput_set(H, W, T, seed=3)
    inds = torch.randint(H * W * T, (B, 1), generator=torch.Generator().manual_seed(2))
    mp, ap = _params(golden_dir)
    vid = A.DeviceVideo.from_reference_layout(data, DEV)
    grads = {}
    for name, prec in (("fp32", N.PREC_FP32), ("tc", N.PREC_TC)):
        tr = A.AtlasTrainer(vid, {"samples_batch": B}, precision=prec, device=DEV)
        tr.load_state(O.state_dict_of(mp), O.state_dict_of(ap))
        tr.indices.copy_(inds.reshape(-1))
        tr.loss_grad(True)
        torch.cuda.synchronize()
        grads[name] = tr.grads.clone()
        if prec == N.PREC_TC:
            cap, x, uv, y = _tc_outputs(tr, B)
            with torch.no_grad():
                uv_ref = O.mlp_forward(O.MAPPING_SPEC, mp, x.cpu()[:, :3])
                y_ref = O.mlp_forward(O.ATLAS_SPEC, ap, uv_ref[:3 * cap] * 0.5 + 0.5)
            live = torch.zeros(9 * cap, dtype=torch.bool)
            cnt = tr.workspace_views()["counters"].cpu()
            for g in range(9):                              # groups 5 / 6 are compacted to the valid flow rows
                live[g * cap:g * cap + (int(cnt[g]) if g in (5, 6) else B)] = True
            assert (uv.cpu() - uv_ref)[live].abs().max() <= 5e-6
            assert (y.cpu() - y_ref)[live[:3 * cap]].abs().max() <= 5e-5
            losses_tc = tr.losses.cpu().numpy().copy()
        else:
            losses_32 = tr.losses.cpu().numpy().copy()
    np.testing.assert_allclose(losses_tc[:6], losses_32[:6], rtol=2e-5)
    # float64 truth
    video64 = O.Video(**{k: v.double() if v.dtype == torch.float32 else v for k, v in data.items()})
    mp64 = [p.double().requires_grad_(True) for p in mp]
    ap64 = [p.double().requires_grad_(True) for p in ap]
    terms = O.iteration_losses(video64, mp64, ap64, inds, 0)
    terms["total"].backward()
    np.testing.assert_allclose(losses_tc[0], float(terms["total"].detach()), rtol=1e-4)
    probe = A.AtlasTrainer(vid, {"samples_batch": B}, precision=N.PREC_FP32, device=DEV)
    truth = [p.grad.float() for p in mp64 + ap64]
    i = 0
    problems = []
    for which in ("mapping", "atlas"):
        g32 = probe._views(grads["fp32"], which)
        gtc = probe._views(grads["tc"], which)
        for k in g32:
            ref = truth[i].to(DEV); i += 1
            e32 = (g32[k] - ref).abs().flatten()
            etc = (gtc[k] - ref).abs().flatten()
            q32 = torch.quantile(e32[:: max(1, e32.numel() // 100000)], 0.9).item()
            qtc = torch.quantile(etc[:: max(1, etc.numel() // 100000)], 0.9).item()
            if qtc > max(10 * q32, 2e-3 * ref.abs().max().item()) + 1e-9:
                problems.append((which, k, "q90", qtc, q32, ref.abs().max().item()))
            if etc.norm().item() > max(3e-3 * ref.norm().item(), 3 * e32.norm().item()) + 1e-9:
                problems.append((which, k, "frobenius", etc.norm().item(), e32.norm().item(), ref.norm().item()))
    assert not problems, problems


def test_tc_trajectory_and_pretrain(golden_dir):
    _need_tc()
    H, W, T, B = 24, 40, 6, 64
    data = synth.throughput_set(H, W, T, seed=3)
    video = O.Video(**data)
    mp, ap = _params(golden_dir)
    vid = A.DeviceVideo.from_reference_layout(data, DEV)
    tr = A.AtlasTrainer(vid, {"samples_batch": B}, precision=N.PREC_TC, device=DEV)
    tr.load_state(O.state_dict_of(mp), O.state_dict_of(ap))
    mp = [p.clone().requires_grad_(True) for p in mp]
    ap = [p.clone().requires_grad_(True) for p in ap]
    opt = O.make_optimizer(mp, ap)
    gi = torch.Generator().manual_seed(21)
    for it in (0, 1, 6000, 6001, 2):                      # both graph variants, interleaved
        inds = torch.randint(H * W * T, (B, 1), generator=gi)
        ref = O.train_iteration(video, mp, ap, opt, inds, it)
        got = tr.step_host(inds, it, use_graph=True)
        np.testing.assert_allclose(got[0], ref["total"], rtol=1e-3)
    for which, ref_p in (("mapping", mp), ("atlas", ap)):
        for (k, v), r in zip(tr.param_views(which).items(), ref_p):
            d = (v.cpu() - r.detach()).abs()
            # 5 Adam steps of lr 1e-4 on an ill-conditioned toy (random-init mapping, 64 samples).  Calibrated with
            # tests/perf/parity_diag.py: max 5.6e-4, mean <= 1.1e-5, <= 14 % of a tensor's entries beyond
            # 2e-5 and <= 1.2 % beyond one learning-rate step.  Bounds = measured x ~2; the well-conditioned,
            # full-size version with tight bounds is tests/test_tc_fullsize_gpu.py.
            assert d.max() <= 1.1e-3, (which, k, float(d.max()))
            assert d.mean() <= 2.5e-5, (which, k, float(d.mean()))
            if d.numel() >= 1000:
                assert d.median() <= 1.2e-5 and (d > 2e-5).float().mean() <= 0.25 and (d > 1e-4).float().mean() <= 0.03, \
                    (which, k, float(d.median()), float((d > 2e-5).float().mean()))
    # pre-training on the tensor-core path
    tr2 = A.AtlasTrainer(vid, {"samples_batch": 10000}, precision=N.PREC_TC, device=DEV)
    mp0, ap0 = _params(golden_dir)
    tr2.load_state(O.state_dict_of(mp0), O.state_dict_of(ap0))
    mpp = [p.clone().requires_grad_(True) for p in mp0]
    torch.manual_seed(5)
    popt = torch.optim.Adam(mpp, lr=1e-4)
    for f in range(2):
        ys = torch.randint(20, (10000, 1)); xs = torch.randint(36, (10000, 1))
        loss = O.pretrain_losses(mpp, f, ys, xs, 2, 36, 0.8)
        popt.zero_grad(); loss.backward(); popt.step()
    torch.manual_seed(5)
    last = tr2.pretrain(2, 20, 36, 1)
    torch.cuda.synchronize()
    np.testing.assert_allclose(float(last[0]), float(loss.detach()), rtol=1e-4)
    for (k, v), r in zip(tr2.param_views("mapping").items(), mpp):
        assert (v.cpu() - r.detach()).abs().max() <= 1e-5, k


def test_tc_render_parity(golden_dir):
    """b200_render with B200_PREC_TC (the fused forward kernels without their image stores) against the oracle's
    render (evaluate.py:640-708): |err| <= 5e-5 on the fp32 image (the atlas-output tolerance above), uint8 frames
    within 1 LSB, PSNR within 1e-3 dB; ragged chunks and a whole-frame call give the same image."""
    _need_tc()
    z = np.load(os.path.join(golden_dir, "iteration.npz"))
    data = {k[6:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("video_")}
    mp, ap = _params(golden_dir)
    H, W, _, T = data["frames"].shape
    vid = A.DeviceVideo.from_reference_layout(data, DEV)
    tr = A.AtlasTrainer(vid, {"samples_batch": 64}, precision=N.PREC_TC, device=DEV)
    tr.load_state(O.state_dict_of(mp), O.state_dict_of(ap))
    before = N.lib().b200_launch_count()
    img, u8 = tr.render_frame(2, H, W, T, want_u8=True)
    assert N.lib().b200_launch_count() - before == 5          # rows, weight images, 2 fused forwards, output
    img_chunks = tr.render_frame(2, H, W, T, chunk=500)
    ref = O.render_frame(mp, ap, 2, H, W, T)
    assert (img.cpu() - ref).abs().max() <= 5e-5
    assert torch.equal(img_chunks, img)
    diff = np.abs(u8.cpu().numpy().astype(int) - O.to_uint8(ref).astype(int))
    assert diff.max() <= 1 and (diff != 0).mean() < 0.01
    assert abs(A.psnr(data["frames"][:, :, :, 2], img.cpu()) - O.psnr(data["frames"][:, :, :, 2], ref)) < 1e-3


@pytest.mark.parametrize("which", ["mapping", "atlas", "mapping4", "alpha"])
def test_imlp_class_on_tensor_cores(golden_dir, which, monkeypatch):
    """The drop-in `IMLP` class (b200_mlp_forward / b200_mlp_backward with B200_PREC_TC) against the oracle network
    with the same parameters: forward |err| <= 5e-6 (mapping) / 5e-5 (atlas, positional-encoding amplification),
    parameter gradients of a random linear functional against FLOAT64: ||err||_F <= 3e-3 ||g||_F per tensor for the
    mapping, 1.5e-2 for the atlas (measured 5.9e-3 on its first layer: the 2^9*pi positional frequency amplifies the
    fp32-level rounding of the encoded input, cf. tests/test_tc_fullsize_gpu.py), input gradient of the atlas likewise.
    rows = 1000: a ragged last tile."""
    _need_tc()
    monkeypatch.setenv("B200_IMLP_PRECISION", "tc")
    from src.models.stage_1.implicit_neural_networks import IMLP
    mp, ap = _params(golden_dir)
    if which == "mapping":
        net = IMLP(input_dim=3, output_dim=2, hidden_dim=256, use_positional=False, positional_dim=4, num_layers=6,
                   skip_layers=[], verbose=False)
        spec, params, scale, tol = O.MAPPING_SPEC, mp, 2.0, 5e-6
    elif which == "mapping4":        # the background mapping of the segmentation variant (4 layers), same kernels
        net = IMLP(input_dim=3, output_dim=2, hidden_dim=256, use_positional=False, positional_dim=2, num_layers=4,
                   skip_layers=[], verbose=False)
        spec = O.MlpSpec(3, 2, 256, False, 2, (), 4)
        torch.manual_seed(77)
        params = O.init_mlp(spec)
        scale, tol = 2.0, 5e-6
    elif which == "alpha":           # the alpha network of the segmentation variant: 3 -> PE 5 -> 256 x 6 -> 1, no skips
        net = IMLP(input_dim=3, output_dim=1, hidden_dim=256, use_positional=True, positional_dim=5, num_layers=8,
                   skip_layers=[], verbose=False)
        spec = O.MlpSpec(3, 1, 256, True, 5, (), 8)
        torch.manual_seed(78)
        params = O.init_mlp(spec)
        scale, tol = 2.0, 2e-5
    else:
        net = IMLP(input_dim=2, output_dim=3, hidden_dim=256, use_positional=True, positional_dim=10, num_layers=8,
                   skip_layers=[4, 7], verbose=False)
        spec, params, scale, tol = O.ATLAS_SPEC, ap, 1.0, 5e-5
    assert net._tc_arch == {"mapping": 1, "mapping4": 1, "atlas": 2, "alpha": 3}[which]
    net.load_state_dict(O.state_dict_of(params))
    net = net.to(DEV)
    g = torch.Generator().manual_seed(4)
    rows = 1000
    x = torch.rand(rows, spec.input_dim, generator=g) * scale - (scale - 1.0)
    w = torch.randn(rows, spec.output_dim, generator=g)
    xd = x.to(DEV).requires_grad_(which == "atlas")
    y = net(xd)
    with torch.no_grad():
        y_ref = O.mlp_forward(spec, params, x)
    assert (y.detach().cpu() - y_ref).abs().max() <= tol
    (y * w.to(DEV)).sum().backward()
    p64 = [p.double().requires_grad_(True) for p in params]
    x64 = x.double().requires_grad_(True)
    (O.mlp_forward(spec, p64, x64) * w.double()).sum().backward()
    views = net._views(net.flat.grad)
    for i in range(len(params) // 2):
        for kind, t in (("weight", p64[2 * i]), ("bias", p64[2 * i + 1])):
            e = (views[f"hidden.{i}.{kind}"].cpu().double() - t.grad).norm() / t.grad.norm()
            assert float(e) <= (1.5e-2 if which == "atlas" else 3e-3), (which, i, kind, float(e))
    print(which, "tensor-core IMLP: forward max err", float((y.detach().cpu() - y_ref).abs().max()))
    if which == "atlas":
        e = (xd.grad.cpu().double() - x64.grad).norm() / x64.grad.norm()
        assert float(e) <= 1.5e-2, float(e)
