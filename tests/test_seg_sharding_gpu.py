"""Frame-sharded segmentation trip on the GPU (`-m gpu`).  The shards of a 2- or 4-way split are evaluated one after
another on one GPU, each with its own DeviceVideo frame block and matte; the SUM of their [gradients || loss vector]
must be the unsharded trip (the formulation tests/test_seg_sharding_gloo.py pins on the CPU).

Tolerances are those of tests/test_seg_gpu.py against oracle/seg_oracle.py: fp32 losses rtol 2e-4, gradients 1e-3
max|grad| per tensor (+ 2e-4 of the network's largest gradient); tensor cores 2e-3 and 1.5e-2 (+ 2e-3)."""
import numpy as np
import pytest
import torch

from b200 import _native as N
from b200 import atlas as A
from b200 import seg as SG
from oracle import atlas_oracle as O
from oracle import seg_oracle as S
from seg_common import ORDER, load_fixture
from test_seg_sharding_gloo import global_flow_counts

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _precisions():
    out = [N.PREC_FP32]
    if torch.cuda.is_available() and N.lib().b200_device_supports_tc():
        out.append(N.PREC_TC)
    return out


def _data(video):
    return dict(frames=video.frames, frames_dx=video.frames_dx, frames_dy=video.frames_dy, flow_fwd=video.flow_fwd,
                flow_bwd=video.flow_bwd, mask_fwd=video.mask_fwd, mask_bwd=video.mask_bwd)


def _shard_trips(data, masks, nets, precision, inds, it, world):
    """[gradients || loss vector] of every rank of a `world`-way frame split, evaluated on this GPU."""
    T = data["frames"].shape[-1]
    out = []
    for r in range(world):
        t0, t1 = A.frame_range(r, world, T)
        vid = A.DeviceVideo.from_reference_layout(data, DEV, t0, t1)
        tr = SG.SegTrainer(vid, SG.pack_mask_frames(masks, DEV, t0, t1), {"samples_batch": inds.shape[0]},
                           precision=precision, device=DEV)
        tr.load_state({k: O.state_dict_of(nets[k]) for k in ORDER})
        tr.indices.copy_(inds.reshape(-1))
        tr.loss_grad(it)
        torch.cuda.synchronize()
        out.append(tr.grad_loss.detach().cpu().double())
    return out, tr


@pytest.mark.parametrize("precision", _precisions())
@pytest.mark.parametrize("world", [2, 4])
@pytest.mark.parametrize("it", [0, 6000])
def test_shard_sum_matches_oracle(golden_dir, world, precision, it):
    z, video, masks, nets = load_fixture(golden_dir)
    inds = torch.from_numpy(z["inds"])
    parts, tr = _shard_trips(_data(video), masks, nets, precision, inds, it, world)
    total = sum(parts)
    got = {k: float(v) for k, v in zip(SG.LOSS_NAMES, total[tr.n_params:])}
    mine = {k: [p.clone().requires_grad_(True) for p in nets[k]] for k in ORDER}
    terms = S.seg_iteration_losses(video, masks, mine, inds, it)
    terms["total"].backward()
    tc = precision == N.PREC_TC
    for k, v in terms.items():
        np.testing.assert_allclose(got[k], float(v.detach()), rtol=2e-3 if tc else 2e-4, err_msg=k)
    n_f, n_b = global_flow_counts(video, inds)
    assert (got["n_fwd"], got["n_bwd"]) == (world * n_f, world * n_b)
    grads = total[:tr.n_params].float()
    for k in ORDER:
        scale_net = max(float(p.grad.abs().max()) for p in mine[k])
        for (name, g), p in zip(tr._views(grads, k).items(), mine[k]):
            bound = (1.5e-2 if tc else 1e-3) * float(p.grad.abs().max()) + (2e-3 if tc else 2e-4) * scale_net + 1e-7
            err = float((g - p.grad).abs().max())
            assert err <= bound, (k, name, err, bound)


@pytest.mark.parametrize("precision", _precisions())
def test_shard_without_samples_adds_nothing(golden_dir, precision):
    """Every sample lies in frame 1 (which has both flow directions), so rank 1 of a 2-way split has no resident
    sample: its networks run on zero live tiles, its gradients are exactly zero and its loss terms zero; the
    whole-batch counts are still there."""
    z, video, masks, nets = load_fixture(golden_dir)
    B = int(z["inds"].shape[0])
    inds = video.H * video.W + torch.randint(video.H * video.W, (B, 1), generator=torch.Generator().manual_seed(11))
    parts, tr = _shard_trips(_data(video), masks, nets, precision, inds, 0, 2)
    empty = parts[1]
    assert torch.count_nonzero(empty[:tr.n_params]) == 0
    losses = empty[tr.n_params:]
    assert torch.all(losses[:12] == 0)
    n_f, n_b = global_flow_counts(video, inds)
    assert n_f > 0 and n_b > 0 and (float(losses[12]), float(losses[13])) == (n_f, n_b)
    assert torch.isfinite(parts[0]).all()


@pytest.mark.parametrize("precision", _precisions())
def test_no_valid_flow_gives_nan_flow_terms(golden_dir, precision):
    """All flow masks zeroed: the flow means are over empty sets (NaN in the reference); the NaN survives the sum over
    ranks as a value while every gradient stays finite."""
    z, video, masks, nets = load_fixture(golden_dir)
    data = _data(video)
    data["mask_fwd"] = torch.zeros_like(data["mask_fwd"])
    data["mask_bwd"] = torch.zeros_like(data["mask_bwd"])
    inds = torch.from_numpy(z["inds"])
    parts, tr = _shard_trips(data, masks, nets, precision, inds, 0, 2)
    total = sum(parts)
    got = {k: float(v) for k, v in zip(SG.LOSS_NAMES, total[tr.n_params:])}
    for k in ("flow1", "flow2", "flow_alpha", "total"):
        assert np.isnan(got[k]), k
    assert got["n_fwd"] == 0 and got["n_bwd"] == 0
    assert torch.isfinite(total[:tr.n_params]).all()


@pytest.fixture
def one_rank_group():
    import os
    import torch.distributed as dist
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", str(29600 + os.getpid() % 1000))
    torch.cuda.set_device(0)
    dist.init_process_group("nccl", rank=0, world_size=1, device_id=torch.device("cuda", 0))
    yield dist.group.WORLD
    dist.destroy_process_group()


@pytest.mark.parametrize("fused", [True, False])
def test_trainer_with_one_rank_group_matches_ungrouped(golden_dir, one_rank_group, fused):
    """Three graph-replayed steps of a SegTrainer with a one-rank NCCL group (fused optimiser over symmetric memory, or
    NCCL all-reduce + local Adam) against the ungrouped trainer on the same index batches.  The exchange and the
    optimiser are bit-exact (test_atlas_gpu::test_dp_adam_single_rank_equals_adam); what may differ is the fp32
    atomic summation order inside the trip, so losses are compared to rtol 1e-4, parameters to 5e-5 (three Adam
    steps of lr 1e-4: the bound of test_seg_gpu's trajectory check) and the Adam moments to 1e-3 of their largest
    entry (the gradient bound of test_seg_gpu; near-cancelling bias gradients differ most)."""
    z, video, masks, nets = load_fixture(golden_dir)
    B = z["traj_inds"].shape[1]
    vid = A.DeviceVideo.from_reference_layout(_data(video), DEV)
    mask = SG.pack_mask_frames(masks, DEV)
    try:
        grouped = SG.SegTrainer(vid, mask, {"samples_batch": B}, device=DEV, process_group=one_rank_group,
                                fused_dp=fused)
    except Exception as e:                      # noqa: BLE001 - symmetric memory unavailable on this machine
        if fused:
            pytest.skip(f"torch symmetric memory unavailable: {type(e).__name__}: {e}")
        raise
    assert (grouped._dp is not None) == fused
    plain = SG.SegTrainer(vid, mask, {"samples_batch": B}, device=DEV)
    for tr in (grouped, plain):
        tr.load_state({k: O.state_dict_of(nets[k]) for k in ORDER})
    for it in range(3):
        a = grouped.step_host(torch.from_numpy(z["traj_inds"][it]), it)
        b = plain.step_host(torch.from_numpy(z["traj_inds"][it]), it)
        np.testing.assert_allclose(a[:12], b[:12], rtol=1e-4)
        assert a[12] == b[12] and a[13] == b[13]
    assert int(grouped.step_count) == int(plain.step_count) == 3
    assert len(grouped._graphs) == 1
    torch.testing.assert_close(grouped.params, plain.params, rtol=0, atol=5e-5)
    sd_g, sd_p = grouped.optimizer_state_dict(), plain.optimizer_state_dict()
    assert sd_g["state"].keys() == sd_p["state"].keys()
    for k in ("exp_avg", "exp_avg_sq"):       # the whole moment buffers, after gather_moments assembled them
        ref = torch.cat([sd_p["state"][i][k].flatten() for i in sd_p["state"]])
        got = torch.cat([sd_g["state"][i][k].flatten() for i in sd_g["state"]])
        torch.testing.assert_close(got, ref, rtol=0, atol=1e-3 * float(ref.abs().max()))


@pytest.mark.parametrize("world", [2, 8])
def test_fullsize_shard_sum_matches_whole_video_trip(world):
    """The benchmark geometry (80 x 432 x 768, 10 000 samples, tensor cores) after one pre-training sweep of both
    mappings: the summed trips of a `world`-way frame split against the whole-video trip on the same batch.  Here every
    shard has many tiles per group, its compacted flow groups have fewer live tiles than its ordinary groups (also the
    alpha batch's groups 3 / 4), and the weight-gradient split runs over partial tile counts.

    Bounds: the fixture's tensor-core bounds (losses rtol 2e-3; gradients 1.5e-2 max|g| per tensor + 2e-3 of the
    network's largest gradient), no looser.  The two sides differ only by fp32 summation order and by each rank's own
    gradient scale for the 2-term fp16 split, the error sources those bounds already cover."""
    if not N.lib().b200_device_supports_tc():
        pytest.skip("needs sm_90")
    from b200 import synth
    T, H, W, B = 80, 432, 768, 10000
    data = synth.throughput_set(H, W, T, seed=0)
    masks = (torch.rand(H, W, T, generator=torch.Generator().manual_seed(2)) < 0.4).float()
    inds = torch.randint(H * W * T, (B, 1), generator=torch.Generator().manual_seed(3))
    # the regime: resident samples and compacted flow rows of every shard, from the host copies of the masks
    t_s = inds.reshape(-1) // (H * W)
    yx = inds.reshape(-1) % (H * W)
    wf = data["mask_fwd"][yx // W, yx % W, t_s, 0] != 0
    tiles = lambda n: (n + 127) // 128
    for r in range(world):
        t0, t1 = A.frame_range(r, world, T)
        here = (t_s >= t0) & (t_s < t1)
        n_loc, n_lf = int(here.sum()), int((here & wf).sum())
        assert tiles(n_loc) >= 5 and tiles(n_lf) < tiles(n_loc) < tiles(B), (r, n_loc, n_lf)
    whole = SG.SegTrainer(A.DeviceVideo.from_reference_layout(data, DEV), SG.pack_mask_frames(masks, DEV), None,
                          precision=N.PREC_TC, device=DEV)
    torch.manual_seed(11)
    whole.init_like_reference()
    for which in ("mapping1", "mapping2"):
        whole.pretrain(which, T, H, W, 1)
    whole.indices.copy_(inds.reshape(-1))
    whole.loss_grad(0)
    torch.cuda.synchronize()
    ref = whole.grad_loss.detach().cpu().double()
    params = whole.params.detach().clone()
    n_params = whole.n_params
    del whole
    torch.cuda.empty_cache()
    total = torch.zeros_like(ref)
    for r in range(world):
        t0, t1 = A.frame_range(r, world, T)
        tr = SG.SegTrainer(A.DeviceVideo.from_reference_layout(data, DEV, t0, t1), SG.pack_mask_frames(masks, DEV, t0, t1),
                           None, precision=N.PREC_TC, device=DEV)
        tr.params.copy_(params)
        tr.indices.copy_(inds.reshape(-1))
        tr.loss_grad(0)
        torch.cuda.synchronize()
        total += tr.grad_loss.detach().cpu().double()
        del tr
        torch.cuda.empty_cache()
    got = dict(zip(SG.LOSS_NAMES, total[n_params:].tolist()))
    want = dict(zip(SG.LOSS_NAMES, ref[n_params:].tolist()))
    for k in SG.LOSS_NAMES[:12]:
        np.testing.assert_allclose(got[k], want[k], rtol=2e-3, err_msg=k)
    assert (got["n_fwd"], got["n_bwd"]) == (world * want["n_fwd"], world * want["n_bwd"])
    shapes = SG.SegTrainer(None, None, None, device=DEV)
    worst = {}
    for k in SG.NETS:
        g_views, r_views = shapes._views(total[:n_params], k), shapes._views(ref[:n_params], k)
        scale_net = max(float(v.abs().max()) for v in r_views.values())
        for name in r_views:
            err = float((g_views[name] - r_views[name]).abs().max())
            bound = 1.5e-2 * float(r_views[name].abs().max()) + 2e-3 * scale_net + 1e-7
            worst[(k, name)] = err / bound
            assert err <= bound, (k, name, err, bound)
    print(f"full-size {world}-way shard sum: worst error / bound {max(worst.values()):.2f}")
