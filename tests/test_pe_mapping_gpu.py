"""Position-encoded mapping networks (use_positional_encoding_mapping1/2: 3 -> PE P -> 256 x {4,2} -> 2) on the GPU,
against the oracle with the mapping's MlpSpec swapped in.  Both precisions where the path has both: the tensor-core
kernels (b200_mlp_tc_architecture 4) and the fp32 CUDA-core kernels.

Tolerances start from the default mapping's tests (tests/test_tc_gpu.py): the encoding of (x, y, t) is computed in
fp32 on both sides from the same fp32 products, so it adds no amplification of its own beyond the higher-frequency
inputs of the first layer; the measured figures are in each test's docstring (H100, this repository's kernels).
"""
import glob
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from b200 import _native as N
from b200 import atlas as A
from b200 import seg as SG
from b200 import synth
from oracle import atlas_oracle as O
from oracle import seg_oracle as S
from seg_common import ORDER, load_fixture

pytestmark = pytest.mark.gpu
DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "all-in-one-deflicker_b200")


def _precisions():
    out = [N.PREC_FP32]
    if torch.cuda.is_available() and N.lib().b200_device_supports_tc():
        out.append(N.PREC_TC)
    return out


def _need_tc():
    if not N.lib().b200_device_supports_tc():
        pytest.skip("no sm_90 device")


def _pe_spec(pe, layers=6):
    return O.MlpSpec(3, 2, 256, True, pe, (), layers)


def _pe_config(pe, batch):
    return {"samples_batch": batch, "use_positional_encoding_mapping1": True, "number_of_positional_encoding_mapping1": pe}


def _atlas_params(golden_dir):
    z = np.load(os.path.join(golden_dir, "params_seed1234.npz"))
    return [torch.from_numpy(z[f"atl{i}"]) for i in range(16)]


def _sorted_rows(x):
    for c in (2, 1, 0):
        x = x[torch.sort(x[:, c], stable=True).indices]
    return x


# _GEOMETRY: the global rigidity offset is 100 pixels; at a larger side of 100 it is 2.0 in normalised coordinates, a
# whole period of every encoding frequency 2^k pi, so a PE mapping's Jacobian over that offset is exactly zero and the
# oracle's autograd of sqrt(|JtJ|^2) at zero is NaN.  The step tests use a 96-pixel-wide video.


def _rel_frobenius(got, ref):
    return float((got.double() - ref).norm() / ref.norm())


# ---------------------------------------------------------------------------------------------------------------------
# (a) the IMLP class
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("layers", [4, 6])
@pytest.mark.parametrize("pe", [2, 4, 10])
def test_imlp_pe_mapping_on_tensor_cores(pe, layers, monkeypatch):
    """IMLP(3, 2, use_positional=True, positional_dim=P, skip_layers=[]) with B200_IMLP_PRECISION=tc, 1000 rows (a
    ragged last tile), inputs in [-1, 1]: forward |err| <= 2e-5 against the fp32 oracle (the alpha network's bound),
    parameter gradients of a random linear functional against FLOAT64, ||err||_F <= 3e-3 ||g||_F per tensor (the
    default mapping's bound).  Measured on an H100: forward <= 2.3e-7; gradients <= 4e-6 where no ReLU mask flips, up
    to 2.8e-3 (P = 2, L = 6, hidden.3.bias) where one pre-activation within rounding of 0 flips its mask (the tests of
    the default mapping explain the mechanism)."""
    _need_tc()
    monkeypatch.setenv("B200_IMLP_PRECISION", "tc")
    from src.models.stage_1.implicit_neural_networks import IMLP
    net = IMLP(input_dim=3, output_dim=2, hidden_dim=256, use_positional=True, positional_dim=pe, num_layers=layers,
               skip_layers=[], verbose=False)
    assert net._tc_arch == 4
    spec = _pe_spec(pe, layers)
    torch.manual_seed(90 + pe + layers)
    params = O.init_mlp(spec)
    net.load_state_dict(O.state_dict_of(params))
    net = net.to(DEV)
    g = torch.Generator().manual_seed(4)
    rows = 1000
    x = torch.rand(rows, 3, generator=g) * 2.0 - 1.0
    w = torch.randn(rows, 2, generator=g)
    y = net(x.to(DEV))
    with torch.no_grad():
        y_ref = O.mlp_forward(spec, params, x)
    fwd = float((y.detach().cpu() - y_ref).abs().max())
    assert fwd <= 2e-5, fwd
    (y * w.to(DEV)).sum().backward()
    p64 = [p.double().requires_grad_(True) for p in params]
    (O.mlp_forward(spec, p64, x.double()) * w.double()).sum().backward()
    views = net._views(net.flat.grad)
    worst = {}
    for i in range(layers):
        for kind, t in (("weight", p64[2 * i]), ("bias", p64[2 * i + 1])):
            e = _rel_frobenius(views[f"hidden.{i}.{kind}"].cpu(), t.grad)
            worst[f"hidden.{i}.{kind}"] = round(e, 6)
            assert e <= 3e-3, (i, kind, e)
    print(f"IMLP PE{pe} L{layers}: forward max err {fwd:.3g}, gradient rel. Frobenius errs {worst}")


# ---------------------------------------------------------------------------------------------------------------------
# (b) the fused single-layer step
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", _precisions())
@pytest.mark.parametrize("it", [0, 6000])
def test_fused_step_with_pe_mapping(golden_dir, precision, it, monkeypatch):
    """One fused step (b200_atlas_loss_grad_for) with a PE-4 mapping, with (it 0) and without (it 6000) the global
    rigidity term, 3000 samples: the sampled coordinate rows and flow-row counts are bit-identical to the default
    mapping's step (sampling does not depend on the mapping); mapping output |err| <= 5e-6 against the fp32 oracle on
    the live rows; total loss and terms within 1e-4 of a FLOAT64 oracle evaluation; per-tensor parameter gradients
    ||err||_F <= 1e-2 ||g||_F against float64.  This toy step (random-init mapping, near-singular rigidity Jacobians) is
    ill-conditioned: measured on an H100, the fp32 path itself is 2.7e-3 (weights) / 4.2e-3 (biases: row sums with
    heavy cancellation) from float64, the tensor-core path 3.2e-3 / 4.9e-3; uv <= 7.5e-8."""
    H, W, T, B = 60, 96, 9, 3000              # not 100 wide: see _GEOMETRY
    data = synth.throughput_set(H, W, T, seed=3)
    inds = torch.randint(H * W * T, (B, 1), generator=torch.Generator().manual_seed(2))
    spec = _pe_spec(4)
    torch.manual_seed(31)
    mp = O.init_mlp(spec)
    ap = _atlas_params(golden_dir)
    vid = A.DeviceVideo.from_reference_layout(data, DEV)
    wg = it <= 5000
    base = A.AtlasTrainer(vid, {"samples_batch": B}, precision=N.PREC_FP32, device=DEV)
    base.indices.copy_(inds.reshape(-1))
    base.loss_grad(wg)
    tr = A.AtlasTrainer(vid, _pe_config(4, B), precision=precision, device=DEV)
    assert tr.map_desc.pe_freqs == 4 and tr.n_params == tr.map_total + tr.atl_total
    tr.load_state(O.state_dict_of(mp), O.state_dict_of(ap))
    tr.indices.copy_(inds.reshape(-1))
    tr.loss_grad(wg)
    torch.cuda.synchronize()
    vb, vt = base.workspace_views(), tr.workspace_views()
    cap = vt["cap"]
    cb, ct = vb["counters"].cpu(), vt["counters"].cpu()
    assert [int(ct[i]) for i in (0, 1, 2, 5, 6)] == [int(cb[i]) for i in (0, 1, 2, 5, 6)]
    live = torch.zeros(9 * cap, dtype=torch.bool)
    n_groups = 9 if wg else 7
    for g in range(n_groups):                                 # groups 5 / 6 are compacted to the valid flow rows
        live[g * cap:g * cap + (int(ct[g]) if g in (5, 6) else B)] = True
    x_b, x_t = vb["x_map"].reshape(9 * cap, 4).cpu(), vt["x_map"].reshape(9 * cap, 4).cpu()
    for g in range(n_groups):
        rows = slice(g * cap, g * cap + (int(ct[g]) if g in (5, 6) else B))
        if g in (5, 6):          # the compacted flow-match groups are filled by atomic slot claims: compare as row sets
            assert torch.equal(_sorted_rows(x_t[rows]), _sorted_rows(x_b[rows])), g
        else:
            assert torch.equal(x_t[rows], x_b[rows]), g
    with torch.no_grad():
        uv_ref = O.mlp_forward(spec, mp, x_t[:, :3])
    uv_err = float((vt["uv"].reshape(9 * cap, 2).cpu() - uv_ref)[live].abs().max())
    assert uv_err <= 5e-6, uv_err
    monkeypatch.setattr(O, "MAPPING_SPEC", spec)
    video64 = O.Video(**{k: v.double() if v.dtype == torch.float32 else v for k, v in data.items()})
    mp64 = [p.double().requires_grad_(True) for p in mp]
    ap64 = [p.double().requires_grad_(True) for p in ap]
    terms = O.iteration_losses(video64, mp64, ap64, inds, it)
    terms["total"].backward()
    losses = tr.losses.cpu().numpy()
    np.testing.assert_allclose(losses[0], float(terms["total"].detach()), rtol=1e-4)
    for idx, name in ((1, "rgb"), (2, "gradient"), (3, "rigidity"), (5, "flow")):
        np.testing.assert_allclose(losses[idx], float(terms[name].detach()), rtol=1e-4, err_msg=name)
    truth = [p.grad for p in mp64 + ap64]
    i, worst = 0, {"weight": 0.0, "bias": 0.0}
    for which in ("mapping", "atlas"):
        for k, g in tr.grad_views(which).items():
            e = _rel_frobenius(g.cpu(), truth[i]); i += 1
            kind = k.rsplit(".", 1)[1]
            worst[kind] = max(worst[kind], e)
            assert e <= 1e-2, (which, k, e)
    print(f"fused step PE4 prec {precision} it {it}: uv err {uv_err:.3g}, worst gradient rel. Frobenius err {worst}")


@pytest.mark.parametrize("precision", _precisions())
def test_pe_mapping_trajectory(golden_dir, precision, monkeypatch):
    """Five graph-replayed Adam steps (both graph variants, interleaved) of the single-layer step with a PE-4 mapping
    against the oracle's train_iteration: loss within 1e-3 each step; parameters after the five steps with the bounds of
    the default mapping's trajectory test (max 1.1e-3, mean 2.5e-5).  Measured on an H100: parameters max 5.3e-4
    (fp32) / 5.0e-4 (tensor cores).  Checkpoint and optimiser state dicts keep the reference's keys and reload."""
    H, W, T, B = 60, 96, 9, 2000              # not 100 wide: see _GEOMETRY
    data = synth.throughput_set(H, W, T, seed=3)
    video = O.Video(**data)
    spec = _pe_spec(4)
    torch.manual_seed(32)
    mp = O.init_mlp(spec)
    ap = _atlas_params(golden_dir)
    vid = A.DeviceVideo.from_reference_layout(data, DEV)
    tr = A.AtlasTrainer(vid, _pe_config(4, B), precision=precision, device=DEV)
    tr.load_state(O.state_dict_of(mp), O.state_dict_of(ap))
    monkeypatch.setattr(O, "MAPPING_SPEC", spec)
    mp = [p.clone().requires_grad_(True) for p in mp]
    ap = [p.clone().requires_grad_(True) for p in ap]
    opt = O.make_optimizer(mp, ap)
    gi = torch.Generator().manual_seed(21)
    for it in (0, 1, 6000, 6001, 2):
        inds = torch.randint(H * W * T, (B, 1), generator=gi)
        ref = O.train_iteration(video, mp, ap, opt, inds, it)
        got = tr.step_host(inds, it, use_graph=True)
        np.testing.assert_allclose(got[0], ref["total"], rtol=1e-3)
    worst = 0.0
    for which, ref_p in (("mapping", mp), ("atlas", ap)):
        for (k, v), r in zip(tr.param_views(which).items(), ref_p):
            d = (v.cpu() - r.detach()).abs()
            worst = max(worst, float(d.max()))
            assert d.max() <= 1.1e-3 and d.mean() <= 2.5e-5, (which, k, float(d.max()), float(d.mean()))
    # checkpoint schema: the reference's keys, the mapping's first layer on the 24 encoding columns
    sd = tr.state_dict("mapping")
    assert len(sd) == 12 and sd["hidden.0.weight"].shape == (256, 24)
    osd = tr.optimizer_state_dict()
    assert len(osd["state"]) == 28 and osd["state"][0]["exp_avg"].shape == (256, 24)
    tr2 = A.AtlasTrainer(vid, _pe_config(4, B), precision=precision, device=DEV)
    tr2.load_state(sd, tr.state_dict("atlas"))
    tr2.load_optimizer_state_dict(osd)
    assert torch.equal(tr2.params, tr.params) and torch.equal(tr2.exp_avg, tr.exp_avg)
    print(f"trajectory PE4 prec {precision}: parameter max diff {worst:.3g}")


# ---------------------------------------------------------------------------------------------------------------------
# (c) render, evaluation maps, pre-training
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", _precisions())
def test_pe_mapping_render_eval_maps_and_pretrain(golden_dir, precision, monkeypatch):
    """render_frame (b200_render_for) against the oracle's render: |err| <= 5e-5 (the default mapping's tensor-core
    bound), uint8 within 1 LSB; chunked and whole-frame renders agree.  eval_maps (b200_eval_maps with the PE mapping):
    uv 5e-6, rigidity / flow error with the default mapping's relative bounds.  Two pre-training steps
    (b200_pretrain_loss_grad_for) against torch Adam on the oracle: loss within 1e-4; parameters max 4e-4 (2 steps x
    2 lr: Adam's early steps are ~lr whatever the gradient's size, so a gradient rounded to opposite signs moves a
    parameter 2 lr apart), mean 2e-7, at most 0.1 % of entries beyond 1e-5.  Measured on an H100 (fp32 / tensor cores):
    render 5.0e-6 / 6.0e-6, uv 3.4e-8 / 8.0e-8, pre-training max 2.2e-5 / 2.6e-4, mean 3.3e-9 / 4.4e-8, beyond 1e-5
    0.002 % / 0.034 %."""
    z = np.load(os.path.join(golden_dir, "iteration.npz"))
    data = {k[6:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("video_")}
    H, W, _, T = data["frames"].shape
    spec = _pe_spec(6)
    torch.manual_seed(33)
    mp = O.init_mlp(spec)
    ap = _atlas_params(golden_dir)
    vid = A.DeviceVideo.from_reference_layout(data, DEV)
    tr = A.AtlasTrainer(vid, _pe_config(6, 64), precision=precision, device=DEV)
    tr.load_state(O.state_dict_of(mp), O.state_dict_of(ap))
    monkeypatch.setattr(O, "MAPPING_SPEC", spec)
    img, u8 = tr.render_frame(2, H, W, T, want_u8=True)
    img_chunks = tr.render_frame(2, H, W, T, chunk=500)
    ref = O.render_frame(mp, ap, 2, H, W, T)
    r_err = float((img.cpu() - ref).abs().max())
    assert r_err <= 5e-5, r_err
    assert torch.equal(img_chunks, img)
    diff = np.abs(u8.cpu().numpy().astype(int) - O.to_uint8(ref).astype(int))
    assert diff.max() <= 1 and (diff != 0).mean() < 0.01
    video = O.Video(**data)
    uv_err = 0.0
    for f in (0, T - 1):
        uv, rig, flow = tr.eval_maps(f, chunk=300)
        uv_r, rig_r, flow_r = O.eval_maps(video, mp, f)
        uv_err = max(uv_err, float((uv.cpu() - uv_r).abs().max()))
        np.testing.assert_allclose(uv.cpu().numpy(), uv_r.numpy(), atol=5e-6)
        np.testing.assert_allclose(rig.cpu().numpy(), rig_r.numpy(), rtol=2e-3, atol=1e-3)
        np.testing.assert_allclose(flow.cpu().numpy(), flow_r.numpy(), rtol=2e-3, atol=2e-4)
    # pre-training of the PE mapping
    tr2 = A.AtlasTrainer(vid, _pe_config(6, 10000), precision=precision, device=DEV)
    tr2.load_state(O.state_dict_of(mp), O.state_dict_of(ap))
    mpp = [p.clone().requires_grad_(True) for p in mp]
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
    # Adam's first steps move a parameter by about lr = 1e-4 whatever its gradient's size, so a gradient that two
    # implementations round to opposite signs puts the parameters up to 2 lr apart per step: the maximum is bounded by
    # 2 steps x 2 lr, the bulk tightly.
    d = torch.cat([(v.cpu() - r.detach()).abs().flatten() for (k, v), r in zip(tr2.param_views("mapping").items(), mpp)])
    p_err, p_mean, p_frac = float(d.max()), float(d.mean()), float((d > 1e-5).float().mean())
    assert p_err <= 4e-4 and p_mean <= 2e-7 and p_frac <= 1e-3, (p_err, p_mean, p_frac)
    print(f"render/eval/pretrain PE6 prec {precision}: render err {r_err:.3g}, eval uv err {uv_err:.3g}, pretrain param diff max {p_err:.3g} "
          f"mean {p_mean:.3g}, beyond 1e-5 {p_frac:.3g}")


# ---------------------------------------------------------------------------------------------------------------------
# (d) the segmentation variant with PE mappings
# ---------------------------------------------------------------------------------------------------------------------
SEG_PE = {"use_positional_encoding_mapping1": True, "number_of_positional_encoding_mapping1": 4,
          "use_positional_encoding_mapping2": True, "number_of_positional_encoding_mapping2": 2}


@pytest.mark.parametrize("it", [0, 6000])
def test_seg_step_with_pe_mappings(golden_dir, it):
    """The segmentation step with PE 4 on mapping1 (6 layers) and PE 2 on mapping2 (4 layers): with B200_PREC_TC both
    mappings run on the tensor cores (code 4).  Against oracle/seg_oracle.py with the same specs: the fp32 path with the
    existing fp32 bounds (losses 2e-4, gradients 1e-3 max|grad|), the tensor-core path with the existing tensor-core
    bounds (losses 2e-3, gradients 1.5e-2 max|grad|); tensor-core losses within 2e-3 of the fp32 path's.  Measured on an
    H100: tensor-core losses <= 7e-6 relative to the oracle."""
    _need_tc()
    z, video, masks, _ = load_fixture(golden_dir)
    specs = dict(mapping1=_pe_spec(4, 6), mapping2=_pe_spec(2, 4), alpha=S.ALPHA_SPEC, atlas=S.ATLAS_SPEC)
    torch.manual_seed(41)
    nets = S.init_nets(specs)
    inds = torch.from_numpy(z["inds"])
    data = dict(frames=video.frames, frames_dx=video.frames_dx, frames_dy=video.frames_dy, flow_fwd=video.flow_fwd,
                flow_bwd=video.flow_bwd, mask_fwd=video.mask_fwd, mask_bwd=video.mask_bwd)
    vid = A.DeviceVideo.from_reference_layout(data, DEV)
    mine = {k: [p.clone().requires_grad_(True) for p in nets[k]] for k in ORDER}
    terms = S.seg_iteration_losses(video, masks, mine, inds, it, specs=specs)
    terms["total"].backward()
    got = {}
    for prec in (N.PREC_FP32, N.PREC_TC):
        tr = SG.SegTrainer(vid, SG.pack_mask_frames(masks, DEV), dict(SEG_PE, samples_batch=inds.shape[0]), precision=prec,
                           device=DEV)
        assert [N.lib().b200_mlp_tc_architecture(tr.descs[k]) for k in ("mapping1", "mapping2")] == [4, 4]
        tr.load_state({k: O.state_dict_of(nets[k]) for k in ORDER})
        tr.indices.copy_(inds.reshape(-1))
        tr.loss_grad(it)
        torch.cuda.synchronize()
        got[prec] = tr.loss_dict()
        tc = prec == N.PREC_TC
        for k, v in terms.items():
            np.testing.assert_allclose(got[prec][k], float(v.detach()), rtol=2e-3 if tc else 2e-4, err_msg=k)
        for k in ORDER:
            scale_net = max(float(p.grad.abs().max()) for p in mine[k])
            for (name, g), p in zip(tr.grad_views(k).items(), mine[k]):
                bound = (1.5e-2 if tc else 1e-3) * float(p.grad.abs().max()) + (2e-3 if tc else 2e-4) * scale_net + 1e-7
                err = float((g.cpu() - p.grad).abs().max())
                assert err <= bound, (prec, k, name, err, bound)
    for k in terms:
        np.testing.assert_allclose(got[N.PREC_TC][k], got[N.PREC_FP32][k], rtol=2e-3, err_msg=k)
    rel = max(abs(got[N.PREC_TC][k] - float(v.detach())) / max(abs(float(v.detach())), 1e-30) for k, v in terms.items())
    print(f"seg step PE mappings it {it}: tensor-core losses max rel err {rel:.3g}")


# ---------------------------------------------------------------------------------------------------------------------
# (e) the single-layer script end to end
# ---------------------------------------------------------------------------------------------------------------------
def _write_video(folder, T=5, H=96, W=128):
    import cv2
    os.makedirs(folder, exist_ok=True)
    rng = np.random.RandomState(1)
    base = cv2.GaussianBlur(rng.rand(H + 32, W + 32, 3).astype(np.float32), (0, 0), 3.0)
    base = (base - base.min()) / (base.max() - base.min())
    for t in range(T):
        crop = base[8 + t:8 + t + H, 4 + 2 * t:4 + 2 * t + W]
        cv2.imwrite(os.path.join(folder, "%05d.png" % t), np.clip(crop * (1.0 + 0.1 * np.sin(t)) * 255.0, 0, 255).astype(np.uint8))


def test_single_layer_script_with_pe_mapping(tmp_path):
    """src/stage1_neural_atlas.py with use_positional_encoding_mapping1: true (4 frequencies) on a tiny synthetic clip:
    the script completes and writes the checkpoint (the mapping's first layer on 24 encoding columns), the output
    frames and the PSNR marker."""
    work, vid = tmp_path, "tinype"
    _write_video(str(work / "data" / "test" / vid))
    cfg = json.load(open(os.path.join(PKG, "src", "config", "config_flow_100.json")))
    cfg.update(iters_num=101, evaluate_every=100, pretrain_iter_number=1, samples_batch=2000, stop_global_rigidity=50,
               use_positional_encoding_mapping1=True, number_of_positional_encoding_mapping1=4)
    cfg_path = str(work / "cfg.json")
    json.dump(cfg, open(cfg_path, "w"))
    env = dict(os.environ, PYTHONPATH=PKG, B200_ALLOW_RANDOM_RAFT="1")    # no pretrained RAFT offline
    r = subprocess.run([sys.executable, os.path.join(PKG, "src", "stage1_neural_atlas.py"), "--vid_name", vid, "--root",
                        "data/test/", "--down", "1", "--config", cfg_path, "--no_artefacts"], cwd=str(work), env=env,
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    res = work / "results" / vid / "stage_1"
    ck = torch.load(str(res / "checkpoint"), weights_only=False)
    assert set(ck) == {"F_atlas_state_dict", "iteration", "model_F_mapping1_state_dict", "optimizer_all_state_dict"}
    assert ck["iteration"] == 100 and ck["model_F_mapping1_state_dict"]["hidden.0.weight"].shape == (256, 24)
    assert len(sorted(glob.glob(str(res / "output" / "*.png")))) == 5
    marker = glob.glob(str(res / "000100" / "PSNR_*"))
    assert len(marker) == 1 and np.isfinite(float(os.path.basename(marker[0])[len("PSNR_"):]))
