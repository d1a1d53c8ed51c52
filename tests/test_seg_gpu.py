"""Parity of the segmentation variant (b200_seg_* through the C ABI) with oracle/seg_oracle.py on the fixture frozen
from the reference's own functions (tests/golden/seg_iteration.npz).  Needs a GPU (`-m gpu`).

Tolerances:
  fp32 path (every network on the CUDA-core kernels): losses rtol 2e-4; parameter gradients |err| <= 1e-3 max|grad|
  per tensor (+ a network-scale floor for near-cancelling bias gradients); network outputs 2e-5.
  tensor-core path (all four networks on wgmma, 2-term fp16 split operands): losses rtol 2e-3;
  gradients 1.5e-2 max|grad| per tensor (the bound of the stand-alone tensor-core IMLP tests).
"""
import numpy as np
import pytest
import torch

from b200 import _native as N
from b200 import atlas as A
from b200 import seg as SG
from oracle import atlas_oracle as O
from oracle import seg_oracle as S
from seg_common import ORDER, load_fixture

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _trainer(z, video, masks, nets, precision, batch):
    data = dict(frames=video.frames, frames_dx=video.frames_dx, frames_dy=video.frames_dy, flow_fwd=video.flow_fwd,
                flow_bwd=video.flow_bwd, mask_fwd=video.mask_fwd, mask_bwd=video.mask_bwd)
    vid = A.DeviceVideo.from_reference_layout(data, DEV)
    tr = SG.SegTrainer(vid, SG.pack_mask_frames(masks, DEV), {"samples_batch": batch}, precision=precision, device=DEV)
    tr.load_state({k: O.state_dict_of(nets[k]) for k in ORDER})
    return tr


def _precisions():
    out = [N.PREC_FP32]
    if torch.cuda.is_available() and N.lib().b200_device_supports_tc():
        out.append(N.PREC_TC)
    return out


def test_param_layout_and_order():
    tr = SG.SegTrainer(None, None, {"samples_batch": 64}, device=DEV)
    assert list(tr.offsets) == ["mapping1", "mapping2", "alpha", "atlas"]
    assert tr.offsets["mapping1"] == 0 and tr.offsets["mapping2"] >= S.MAPPING1_SPEC.num_params()
    assert N.lib().b200_mlp_tc_architecture(tr.descs["mapping1"]) == 1
    assert N.lib().b200_mlp_tc_architecture(tr.descs["mapping2"]) == 1      # 4-layer mapping: same tensor-core kernels
    assert N.lib().b200_mlp_tc_architecture(tr.descs["alpha"]) == 3         # PE 5 / one output: the alpha variant
    assert N.lib().b200_mlp_tc_architecture(tr.descs["atlas"]) == 2
    torch.manual_seed(int(4321))
    tr.init_like_reference()
    torch.manual_seed(int(4321))
    nets = S.init_nets()
    for k in ORDER:
        for (name, v), p in zip(tr.param_views(k).items(), nets[k]):
            assert torch.equal(v.cpu(), p), (k, name)


@pytest.mark.parametrize("precision", _precisions())
@pytest.mark.parametrize("it", [0, 6000, 10001])
def test_seg_iteration_matches_oracle(golden_dir, it, precision):
    z, video, masks, nets = load_fixture(golden_dir)
    inds = torch.from_numpy(z["inds"])
    tr = _trainer(z, video, masks, nets, precision, inds.shape[0])
    tr.indices.copy_(inds.reshape(-1))
    tr.loss_grad(it)
    torch.cuda.synchronize()
    got = tr.loss_dict()
    mine = {k: [p.clone().requires_grad_(True) for p in nets[k]] for k in ORDER}
    terms = S.seg_iteration_losses(video, masks, mine, inds, it)
    terms["total"].backward()
    tc = precision == N.PREC_TC
    for k, v in terms.items():
        np.testing.assert_allclose(got[k], float(v.detach()), rtol=2e-3 if tc else 2e-4, err_msg=k)
    if it > 5000:
        assert got["rigidity_global1"] == 0 and got["rigidity_global2"] == 0
    tag = f"it{it}_"
    np.testing.assert_allclose(got["total"], float(z[tag + "loss_total"]), rtol=2e-3 if tc else 2e-4)
    for k in ORDER:
        scale_net = max(float(p.grad.abs().max()) for p in mine[k])
        for (name, g), p in zip(tr.grad_views(k).items(), mine[k]):
            ref = p.grad
            bound = (1.5e-2 if tc else 1e-3) * float(ref.abs().max()) + (2e-3 if tc else 2e-4) * scale_net + 1e-7
            err = float((g.cpu() - ref).abs().max())
            assert err <= bound, (k, name, err, bound)


@pytest.mark.parametrize("precision", _precisions())
def test_seg_trajectory_and_render(golden_dir, precision):
    z, video, masks, nets = load_fixture(golden_dir)
    B = z["traj_inds"].shape[1]
    tr = _trainer(z, video, masks, nets, precision, B)
    keys = [str(k) for k in z["traj_keys"]]
    tc = precision == N.PREC_TC
    for it in range(3):
        out = tr.step_host(torch.from_numpy(z["traj_inds"][it]), it)
        got = tr.loss_dict(out)
        np.testing.assert_allclose([got[k] for k in keys], z["traj_losses"][it], rtol=5e-3 if tc else 5e-4)
    assert int(tr.step_count) == 3
    assert len(tr._graphs) == 1                      # the three trips replayed one captured graph
    # the same three trips launched eagerly (no graph) give the same losses up to atomic summation order
    tr2 = _trainer(z, video, masks, nets, precision, B)
    for it in range(3):
        tr2.indices.copy_(torch.from_numpy(z["traj_inds"][it]).reshape(-1))
        tr2.step(it, use_graph=False)
    torch.cuda.synchronize()
    eager, replay = tr2.loss_dict(), tr.loss_dict()
    for k in keys:
        np.testing.assert_allclose(replay[k], eager[k], rtol=2e-3 if tc else 2e-4, err_msg=k)
    for k in ORDER:
        head = tr.param_views(k)["hidden.0.weight"].flatten()[:64].cpu().numpy()
        # three Adam steps move every weight by <= 3e-4; the sign pattern of the first steps is what can differ
        np.testing.assert_allclose(head, z[f"traj_{k}_head"], rtol=0, atol=(2.5e-4 if tc else 5e-5))
    img, alpha = tr.render_frame(int(z["render_frame"]), video.H, video.W, video.T)
    np.testing.assert_allclose(alpha.cpu().numpy(), z["render_alpha"], atol=2e-3 if tc else 2e-4)
    np.testing.assert_allclose(img.cpu().numpy(), z["render_img"], atol=5e-3 if tc else 5e-4)
    # checkpoint schema of evaluate.py:216-223
    sd = tr.optimizer_state_dict()
    n_tensors = sum(2 * s.num_layers for s in (S.MAPPING1_SPEC, S.MAPPING2_SPEC, S.ALPHA_SPEC, S.ATLAS_SPEC))
    assert len(sd["state"]) == n_tensors and len(sd["param_groups"]) == 4
    assert sd["param_groups"][1]["params"][0] == 2 * S.MAPPING1_SPEC.num_layers


def test_render_of_fixture_parameters_exact_inputs(golden_dir):
    """fp32 reconstruction of the initial parameters against the oracle's render (same composite arithmetic)."""
    z, video, masks, nets = load_fixture(golden_dir)
    tr = _trainer(z, video, masks, nets, N.PREC_FP32, 64)
    img, alpha, u8 = tr.render_frame(2, video.H, video.W, video.T, chunk=500, want_u8=True)
    ref_img, ref_alpha = S.render_frame_seg(nets, 2, video.H, video.W, video.T)
    np.testing.assert_allclose(alpha.cpu().numpy(), ref_alpha.numpy(), atol=2e-5)
    np.testing.assert_allclose(img.cpu().numpy(), ref_img.numpy(), atol=2e-5)
    assert np.abs(u8.cpu().numpy().astype(int) - O.to_uint8(ref_img).astype(int)).max() <= 1


@pytest.mark.parametrize("which", ["mapping1", "mapping2"])
def test_seg_pretrain_matches_oracle(golden_dir, which):
    """pre_train_mapping of either mapping network: one sweep over 2 frames, same index stream as the oracle loop."""
    z, video, masks, nets = load_fixture(golden_dir)
    tr = _trainer(z, video, masks, nets, N.PREC_FP32, 64)
    spec = S.MAPPING1_SPEC if which == "mapping1" else S.MAPPING2_SPEC
    Hp, Wp, Tp = 20, 36, 2
    mp = [p.clone().requires_grad_(True) for p in nets[which]]
    opt = torch.optim.Adam(mp, lr=1e-4)
    torch.manual_seed(5)
    want = []
    for f in range(Tp):
        ys = torch.randint(Hp, (10000, 1)); xs = torch.randint(Wp, (10000, 1))
        i_s, j_s = ys / O._half(max(Wp, Hp)) - 1, xs / O._half(max(Wp, Hp)) - 1
        xyt = torch.cat((j_s, i_s, (f / (Tp / 2.0) - 1) * torch.ones_like(i_s)), dim=1)
        loss = (xyt[:, :2] * 0.8 - O.mlp_forward(spec, mp, xyt)).norm(dim=1).mean()
        opt.zero_grad(); loss.backward(); opt.step()
        want.append(float(loss.detach()))
    torch.manual_seed(5)
    last = tr.pretrain(which, Tp, Hp, Wp, 1)
    np.testing.assert_allclose(float(last), want[-1], rtol=2e-4)
    for (name, v), p in zip(tr.param_views(which).items(), mp):
        np.testing.assert_allclose(v.cpu().numpy(), p.detach().numpy(), rtol=0, atol=5e-5, err_msg=name)
    other = "mapping2" if which == "mapping1" else "mapping1"
    for (name, v), p in zip(tr.param_views(other).items(), nets[other]):
        assert torch.equal(v.cpu(), p), name           # the other networks are untouched
