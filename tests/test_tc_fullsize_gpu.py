"""The tensor-core path (B200_PREC_TC) — the one bench.py times — against the oracle AT THE BENCHMARKED
CONFIGURATION: 80 frames of 432x768, 10 000 samples per iteration (BASELINE.json configs[1]).

Scenario A, throughput set (i.i.d. noise video, random-init networks: what bench.py runs):
  * sampled coordinate rows, gathered targets, flow-row counts           bit-exact
  * the six loss values against the fp32 oracle                          rtol 2e-4
  * every parameter gradient against a FLOAT64 evaluation of the oracle  ||err||_F <= 8e-2 ||g||_F and
    max|err| <= 0.12 max|g| per tensor (0.3 for the two-element mapping output bias, a near-cancelling sum).
    The random-init mapping makes the rigidity Jacobians singular (JtJ ~ 0, 1e-3 regulariser, loss ~1e3 per
    sample), so the gradient is ill-conditioned with respect to fp32 rounding of uv: the fp32 CPU oracle itself
    is 1e-3 ... 1e-2 away from float64 on this input.  These are absolute bounds on that hard case.
Scenario B, quality set (smooth flickering translation) with the mapping pre-trained for two sweeps on the GPU
(J ~ 0.8 I, the state the main loop actually runs in):
  * losses rtol 2e-5; gradients against float64: ||err||_F <= 2.5e-2 ||g||_F and max|err| <= 2.5e-2 max|g|
    per tensor (measured worst 7.1e-3 / 6.5e-3 in the calibration run; the two GPU pre-training sweeps that produce the
    state are themselves not bit-reproducible, and one of ~15 runs exceeded 1.5e-2 / the trajectory bounds below at half
    their present values: the 2^9*pi positional frequency of the atlas turns the 1e-7 uv
    rounding of ANY fp32 forward into 1e-4-relative colour gradients; the fp32 oracle sits at 1.6e-3)
  * 5 Adam steps from that state, same index batches as the oracle: total loss within 6e-4 relative at every
    step (measured 8.6e-5); Adam first moments ||m - m_ref||_F <= 0.2 ||m_ref||_F per tensor (measured 4.2e-2);
    parameters: mean |d| <= 4e-5 and at most 6 % of the entries of a tensor further than one learning-rate step (1e-4)
    from the oracle's (measured 1.2 %).
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
H, W, T, B = 432, 768, 80, 10000
KEYS = ("total", "rgb", "gradient", "rigidity", "rigidity_global", "flow")


def _need_tc():
    if not N.lib().b200_device_supports_tc():
        pytest.skip("no sm_90 device")


def _params(golden_dir):
    z = np.load(os.path.join(golden_dir, "params_seed1234.npz"))
    return ([torch.from_numpy(z[f"map{i}"]) for i in range(12)], [torch.from_numpy(z[f"atl{i}"]) for i in range(16)])


def _truth64(data, mp, ap, inds, it):
    video64 = O.Video(**{k: v.double() if v.dtype == torch.float32 else v for k, v in data.items()})
    m64 = [p.double().requires_grad_(True) for p in mp]
    a64 = [p.double().requires_grad_(True) for p in ap]
    terms = O.iteration_losses(video64, m64, a64, inds, it)
    terms["total"].backward()
    return [p.grad for p in m64 + a64]


def _grad_errors(tr, truth):
    out, i = [], 0
    for which in ("mapping", "atlas"):
        for k, g in tr.grad_views(which).items():
            t = truth[i]; i += 1
            e = (g.cpu().double() - t).abs()
            out.append((f"{which}.{k}", float(e.norm() / t.norm()), float(e.max() / t.abs().max())))
    return out


@pytest.fixture(scope="module")
def inds():
    return torch.randint(H * W * T, (B, 1), generator=torch.Generator().manual_seed(1))


@pytest.mark.parametrize("with_global,it", [(True, 0), (False, 6000)])
def test_throughput_set_sampling_losses_gradients(golden_dir, inds, with_global, it):
    _need_tc()
    torch.set_num_threads(min(32, os.cpu_count() or 1))
    data = synth.throughput_set(H, W, T, seed=0)
    mp, ap = _params(golden_dir)
    vid = A.DeviceVideo.from_reference_layout(data, DEV)
    tr = A.AtlasTrainer(vid, {"samples_batch": B}, precision=N.PREC_TC, device=DEV)
    tr.load_state(O.state_dict_of(mp), O.state_dict_of(ap))
    tr.indices.copy_(inds.reshape(-1))
    tr.loss_grad(with_global)
    torch.cuda.synchronize()
    losses = tr.losses.cpu().numpy()
    # ---- sampling: bit-exact
    video = O.Video(**data)
    jif = O.pixel_table(T, H, W)[:, inds]
    wf = video.mask_fwd[jif[1].squeeze(), jif[0].squeeze(), jif[2].squeeze(), 0] != 0
    wb = video.mask_bwd[jif[1].squeeze(), jif[0].squeeze(), jif[2].squeeze(), 0] != 0
    view = tr.workspace_views()
    assert view["counters"][:3].tolist() == [B, int(wf.sum()), int(wb.sum())]
    assert losses[6] == int(wf.sum()) and losses[7] == int(wb.sum())
    x_map = view["x_map"].cpu()
    assert torch.equal(x_map[0, :B, :3], O.normalise_xyt(jif, max(W, H), T))
    hl = O._half(max(W, H))
    ymd = torch.cat((jif[0] / hl - 1, (jif[1] - 1) / hl - 1, jif[2] / (T / 2.0) - 1), dim=1)
    assert torch.equal(x_map[3, :B, :3], ymd)
    tg = view["targets"].cpu()
    assert torch.equal(tg[:B, 0:3], video.frames[jif[1], jif[0], :, jif[2]].squeeze(1))
    assert torch.equal(tg[:B, 3:6], video.frames_dx[jif[1], jif[0], :, jif[2]].squeeze(1))
    # ---- losses against the fp32 oracle
    with torch.no_grad():
        t32 = O.iteration_losses(video, mp, ap, inds, it)
    ref = [float(t32[k]) if k in t32 else 0.0 for k in KEYS]
    np.testing.assert_allclose(losses[:6], ref, rtol=2e-4)
    # ---- gradients against float64
    bad = []
    for name, fro, mx in _grad_errors(tr, _truth64(data, mp, ap, inds, it)):
        lim_f, lim_m = (0.3, 0.3) if name == "mapping.hidden.5.bias" else (8e-2, 0.12)
        if fro > lim_f or mx > lim_m:
            bad.append((name, fro, mx))
    assert not bad, bad


def test_trained_state_gradients_and_trajectory(golden_dir, inds):
    _need_tc()
    torch.set_num_threads(min(32, os.cpu_count() or 1))
    data = synth.quality_set(H, W, T, seed=0)
    data.pop("clean")
    mp, ap = _params(golden_dir)
    vid = A.DeviceVideo.from_reference_layout(data, DEV)
    tr = A.AtlasTrainer(vid, {"samples_batch": B}, precision=N.PREC_TC, device=DEV)
    tr.load_state(O.state_dict_of(mp), O.state_dict_of(ap))
    torch.manual_seed(11)
    tr.pretrain(T, H, W, 2)
    mq = [v.detach().cpu().clone() for v in tr.param_views("mapping").values()]
    aq = [v.detach().cpu().clone() for v in tr.param_views("atlas").values()]
    video = O.Video(**data)
    for wg, it in ((True, 0), (False, 6000)):
        tr.indices.copy_(inds.reshape(-1)); tr.loss_grad(wg); torch.cuda.synchronize()
        with torch.no_grad():
            t32 = O.iteration_losses(video, mq, aq, inds, it)
        ref = [float(t32[k]) if k in t32 else 0.0 for k in KEYS]
        np.testing.assert_allclose(tr.losses.cpu().numpy()[:6], ref, rtol=2e-5)
        bad = [(n, f, m) for n, f, m in _grad_errors(tr, _truth64(data, mq, aq, inds, it)) if f > 2.5e-2 or m > 2.5e-2]
        assert not bad, (wg, bad)
    # ---- five Adam steps side by side with the oracle
    rm = [p.clone().requires_grad_(True) for p in mq]
    ra = [p.clone().requires_grad_(True) for p in aq]
    opt = O.make_optimizer(rm, ra)
    gi = torch.Generator().manual_seed(21)
    for it in range(5):
        ii = torch.randint(H * W * T, (B, 1), generator=gi)
        ref = O.train_iteration(video, rm, ra, opt, ii, it)
        got = tr.step_host(ii, it)
        assert abs(got[0] - ref["total"]) <= 6e-4 * abs(ref["total"]), (it, got[0], ref["total"])
    bad = []
    for which, ref_p in (("mapping", rm), ("atlas", ra)):
        m_views = tr._views(tr.exp_avg, which)
        for (k, pv), r in zip(tr.param_views(which).items(), ref_p):
            d = (pv.cpu() - r.detach()).abs()
            st = opt.state[r]
            m_err = float((m_views[k].cpu() - st["exp_avg"]).norm() / st["exp_avg"].norm())
            far = float((d > 1e-4).float().mean())
            if m_err > 0.2 or float(d.mean()) > 4e-5 or far > 0.06 or float(d.max()) > 1.1e-3:
                bad.append((which, k, m_err, float(d.mean()), far, float(d.max())))
    assert not bad, bad
