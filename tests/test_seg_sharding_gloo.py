"""N>1 host logic of the segmentation variant on CPU (gloo, world_size 2 and 4): the frame-sharded formulation the
CUDA trip implements.  Every rank sees the same index batch, keeps the samples whose frame it owns, normalises every
mean by the GLOBAL batch and every flow mean by the GLOBAL valid-row counts, and one SUM all-reduce of
(gradients || loss vector) reproduces the unsharded iteration of oracle/seg_oracle.py.  The count entries are the
global counts on every rank, so they read world * count after the sum.  tests/test_seg_sharding_gpu.py checks the
CUDA trip against the same formulation."""
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from b200 import atlas as A
from oracle import atlas_oracle as O
from oracle import seg_oracle as S
from seg_common import load_fixture

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
NETS = ("mapping1", "mapping2", "alpha", "atlas")               # flat-buffer order of SegTrainer
TERMS = ("total", "rgb", "gradient", "sparsity", "rigidity1", "rigidity2", "rigidity_global1", "rigidity_global2",
         "flow1", "flow2", "flow_alpha", "bootstrapping")
MEANS = ("rgb", "gradient", "sparsity", "rigidity1", "rigidity2", "rigidity_global1", "rigidity_global2",
         "bootstrapping")
IT = 0                                                          # global rigidity and bootstrapping both on


def _total(t, cfg=S.SEG_CONFIG):
    """The weighting of stage1_neural_atlas_seg.py:309-315 (seg_oracle.seg_iteration_losses) at IT."""
    return (cfg["rigidity_coeff"] * (t["rigidity1"] + t["rigidity2"])
            + cfg["global_rigidity_coeff_fg"] * t["rigidity_global1"] + cfg["global_rigidity_coeff_bg"] * t["rigidity_global2"]
            + cfg["rgb_coeff"] * t["rgb"] + cfg["optical_flow_coeff"] * (t["flow1"] + t["flow2"])
            + cfg["alpha_bootstrapping_factor"] * t["bootstrapping"] + cfg["alpha_flow_factor"] * t["flow_alpha"]
            + cfg["sparsity_coeff"] * t["sparsity"] + cfg["gradient_loss_coeff"] * t["gradient"])


def global_flow_counts(video, inds):
    H, W, T = video.H, video.W, video.T
    jif = O.pixel_table(T, H, W)[:, inds]
    n_f = int((video.mask_fwd[jif[1].squeeze(), jif[0].squeeze(), jif[2].squeeze(), 0] != 0).sum())
    n_b = int((video.mask_bwd[jif[1].squeeze(), jif[0].squeeze(), jif[2].squeeze(), 0] != 0).sum())
    return n_f, n_b


def sharded_terms(video, masks, nets, inds, t0, t1):
    """This rank's share of every seg loss term: the samples of frames [t0, t1), normalised by global counts."""
    H, W, T = video.H, video.W, video.T
    B = inds.shape[0]
    n_f, n_b = global_flow_counts(video, inds)
    t_all = O.pixel_table(T, H, W)[2, inds.reshape(-1)]
    sub = inds[(t_all >= t0) & (t_all < t1)]
    zero = sum(p.sum() * 0 for k in NETS for p in nets[k])
    if sub.shape[0] == 0:
        return {k: zero for k in TERMS[1:]}
    # the per-sample means of seg_oracle.seg_iteration_losses over this rank's samples, scaled by n_local / B
    cfg = S.SEG_CONFIG
    larger = max(W, H)
    s, d = cfg["uv_mapping_scale"], cfg["derivative_amount"]
    net = lambda k: (lambda x: O.mlp_forward(getattr(S, k.upper() + "_SPEC"), nets[k], x))
    mapping1, mapping2, alpha_net, atlas = net("mapping1"), net("mapping2"), net("alpha"), net("atlas")
    jif = O.pixel_table(T, H, W)[:, sub]
    rgb = video.frames[jif[1], jif[0], :, jif[2]].squeeze(1)
    a_gt = masks[jif[1], jif[0], jif[2]].squeeze(1).unsqueeze(-1)
    xyt = O.normalise_xyt(jif, larger, T)
    uv1, uv2 = mapping1(xyt), mapping2(xyt)
    alpha = S.alpha_of(alpha_net(xyt))
    rgb1 = (atlas(uv1 * 0.5 + 0.5) + 1.0) * 0.5
    rgb2 = (atlas(uv2 * 0.5 - 0.5) + 1.0) * 0.5
    rgb_out = rgb1 * alpha + rgb2 * (1.0 - alpha)
    local = dict(
        gradient=S.gradient_loss_seg(video, jif, mapping1, mapping2, atlas, alpha_net, rgb_out, W),
        rgb=(torch.norm(rgb_out - rgb, dim=1) ** 2).mean(),
        sparsity=(torch.norm(rgb1 * (1.0 - alpha), dim=1) ** 2).mean(),
        rigidity1=O.rigidity_loss(jif, d, larger, T, mapping1, uv1, uv_scale=s),
        rigidity2=O.rigidity_loss(jif, d, larger, T, mapping2, uv2, uv_scale=s),
        rigidity_global1=O.rigidity_loss(jif, cfg["global_rigidity_derivative_amount_fg"], larger, T, mapping1, uv1,
                                         uv_scale=s),
        rigidity_global2=O.rigidity_loss(jif, cfg["global_rigidity_derivative_amount_bg"], larger, T, mapping2, uv2,
                                         uv_scale=s),
        bootstrapping=torch.mean(-a_gt * torch.log(alpha) - (1 - a_gt) * torch.log(1 - alpha)))
    out = {k: local[k] * (sub.shape[0] / B) for k in MEANS}
    # flow terms: sums over this rank's valid rows over the global counts (seg_oracle.flow_loss_alpha /
    # flow_alpha_loss with the two means split open); a direction without valid rows here adds nothing
    def valid(fwd):
        m = video.mask_fwd if fwd else video.mask_bwd
        return bool((m[jif[1].squeeze(), jif[0].squeeze(), jif[2].squeeze(), 0] != 0).any())

    def matches(fwd, values):
        return O.flow_matches(jif, video.mask_fwd if fwd else video.mask_bwd, video.flow_fwd if fwd else video.flow_bwd,
                              larger, T, fwd, values)

    def flow_term(mapping, uv, weight):
        sums = []
        for fwd in (True, False):
            if not valid(fwd):
                sums.append(zero)
                continue
            uv_m, xyt_m, rows = matches(fwd, uv)
            l = (mapping(xyt_m) - uv_m).norm(dim=1) * larger / (2 * s)
            sums.append((l * weight[rows].reshape(-1)).sum())
        return 0.5 * sums[0] / n_f + 0.5 * sums[1] / n_b

    out["flow1"] = flow_term(mapping1, uv1, alpha)
    out["flow2"] = flow_term(mapping2, uv2, 1 - alpha)
    sums = []
    for fwd in (True, False):
        if not valid(fwd):
            sums.append(zero)
            continue
        _, xyt_m, rows = matches(fwd, alpha)
        sums.append((alpha[rows] - S.alpha_of(alpha_net(xyt_m))).abs().sum())
    out["flow_alpha"] = 0.5 * sums[0] / n_f + 0.5 * sums[1] / n_b
    return out


def _worker(rank, world, port, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.set_num_threads(1)
    z, video, masks, nets = load_fixture(GOLDEN)
    nets = {k: [p.clone().requires_grad_(True) for p in nets[k]] for k in NETS}
    inds = torch.from_numpy(z["inds"])
    t0, t1 = A.frame_range(rank, world, video.T)
    terms = sharded_terms(video, masks, nets, inds, t0, t1)
    total = _total(terms)
    total.backward()
    n_f, n_b = global_flow_counts(video, inds)
    flat = torch.cat([p.grad.flatten() if p.grad is not None else torch.zeros(p.numel()) for k in NETS for p in nets[k]]
                     + [torch.stack([total.detach()] + [terms[k].detach() for k in TERMS[1:]]),
                        torch.tensor([float(n_f), float(n_b)])])
    dist.all_reduce(flat)                     # ONE collective: gradients || losses
    if rank == 0:
        q.put(flat.numpy())
    dist.destroy_process_group()


@pytest.mark.timeout(300)
@pytest.mark.parametrize("world", [2, 4])
def test_seg_frame_sharding_reproduces_single_rank(world):
    """world 4 on the 6-frame fixture gives ragged frame blocks (2, 2, 1, 1 frames)."""
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 31500 + (os.getpid() % 2000) + 7 * world
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs: p.start()
    got = q.get(timeout=240)
    for p in procs: p.join(60)
    assert all(p.exitcode == 0 for p in procs)
    z, video, masks, nets = load_fixture(GOLDEN)
    nets = {k: [p.clone().requires_grad_(True) for p in nets[k]] for k in NETS}
    inds = torch.from_numpy(z["inds"])
    terms = S.seg_iteration_losses(video, masks, nets, inds, IT)
    terms["total"].backward()
    ref = torch.cat([p.grad.flatten() for k in NETS for p in nets[k]]).numpy()
    n = ref.size
    assert np.abs(got[:n] - ref).max() <= 2e-4 * np.abs(ref).max()
    np.testing.assert_allclose(got[n:n + len(TERMS)], [float(terms[k].detach()) for k in TERMS], rtol=2e-4)
    n_f, n_b = global_flow_counts(video, inds)
    assert got[n + len(TERMS):].tolist() == [world * n_f, world * n_b]
