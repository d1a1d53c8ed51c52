"""CPU restatement (oracle) of the segmentation variant of the stage-1 loop
(src/stage1_neural_atlas_seg.py:127-315 of the reference): two mapping networks (foreground /
background), an alpha network, one atlas network sampled in two quadrants, and the loss terms
that only this variant has.

TEST INFRASTRUCTURE ONLY — same rule as oracle/atlas_oracle.py: imported by ``tests/``,
``__graft_entry__.smoke()`` and ``bench.py``'s CPU legs, never by the product.

Parity pinning: ``tests/golden/make_golden_seg.py`` runs the reference's own
``get_gradient_loss`` / ``get_rigidity_loss`` / ``get_optical_flow_loss(use_alpha=True)`` /
``get_optical_flow_alpha_loss`` and its ``IMLP`` (imported from /root/reference in the build
container) on the same inputs, asserts bit-equality with the functions below and freezes
``tests/golden/seg_iteration.npz``; ``tests/test_seg_oracle_golden.py`` replays it.
"""
from __future__ import annotations

from typing import Dict, Sequence

import numpy as np
import torch

from oracle import atlas_oracle as O
from oracle.atlas_oracle import MlpSpec, _half

# the four networks of the script with src/config/config_flow_100.json (stage1_neural_atlas_seg.py:127-161)
MAPPING1_SPEC = MlpSpec(3, 2, 256, False, 4, (), 6)
MAPPING2_SPEC = MlpSpec(3, 2, 256, False, 2, (), 4)
ATLAS_SPEC = MlpSpec(2, 3, 256, True, 10, (4, 7), 8)
ALPHA_SPEC = MlpSpec(3, 1, 256, True, 5, (), 8)

SEG_CONFIG = dict(rgb_coeff=5000, optical_flow_coeff=500.0, gradient_loss_coeff=1000, rigidity_coeff=1.0,
                  derivative_amount=1, uv_mapping_scale=0.8, alpha_bootstrapping_factor=2000.0,
                  alpha_flow_factor=4900.0, sparsity_coeff=1000.0, stop_bootstrapping_iteration=10000,
                  global_rigidity_derivative_amount_fg=100, global_rigidity_derivative_amount_bg=100,
                  global_rigidity_coeff_fg=5.0, global_rigidity_coeff_bg=50.0, stop_global_rigidity=5000,
                  samples_batch=10000, iters_num=10001, pretrain_iter_number=100)


def alpha_of(raw: torch.Tensor) -> torch.Tensor:
    """tanh output -> (0.001, 0.991): stage1_neural_atlas_seg.py:226-229 (three separate roundings)."""
    a = 0.5 * (raw + 1.0)
    a = a * 0.99
    return a + 0.001


def gradient_loss_seg(video: O.Video, jif, mapping1, mapping2, atlas, alpha_net, rgb_out, resx: int):
    """``get_gradient_loss`` loss_utils.py:173-224 (two layers + alpha)."""
    T = video.T
    xp = torch.cat(((jif[0] + 1) / _half(resx) - 1, jif[1] / _half(resx) - 1, jif[2] / (T / 2.0) - 1), dim=1)
    yp = torch.cat((jif[0] / _half(resx) - 1, (jif[1] + 1) / _half(resx) - 1, jif[2] / (T / 2.0) - 1), dim=1)
    a_xp = alpha_of(alpha_net(xp))
    a_yp = alpha_of(alpha_net(yp))
    dx_gt = video.frames_dx[jif[1], jif[0], :, jif[2]].squeeze(1)
    dy_gt = video.frames_dy[jif[1], jif[0], :, jif[2]].squeeze(1)
    uv2_yp, uv2_xp = mapping2(yp), mapping2(xp)
    uv1_yp, uv1_xp = mapping1(yp), mapping1(xp)
    rgb1_yp = (atlas(uv1_yp * 0.5 + 0.5) + 1.0) * 0.5
    rgb1_xp = (atlas(uv1_xp * 0.5 + 0.5) + 1.0) * 0.5
    rgb2_yp = (atlas(uv2_yp * 0.5 - 0.5) + 1.0) * 0.5
    rgb2_xp = (atlas(uv2_xp * 0.5 - 0.5) + 1.0) * 0.5
    out_yp = rgb1_yp * a_yp + rgb2_yp * (1.0 - a_yp)
    out_xp = rgb1_xp * a_xp + rgb2_xp * (1.0 - a_xp)
    dx_out = out_xp - rgb_out
    dy_out = out_yp - rgb_out
    return torch.mean((dx_gt - dx_out).norm(dim=1) ** 2 + (dy_gt - dy_out).norm(dim=1) ** 2)


def flow_loss_alpha(video: O.Video, jif, uv, resx, mapping, uv_scale: float, alpha):
    """``get_optical_flow_loss(use_alpha=True)`` loss_utils.py:299-322."""
    T = video.T
    uv_f, xyt_f, rows_f = O.flow_matches(jif, video.mask_fwd, video.flow_fwd, resx, T, True, uv)
    l_next = (mapping(xyt_f) - uv_f).norm(dim=1) * resx / (2 * uv_scale)
    uv_b, xyt_b, rows_b = O.flow_matches(jif, video.mask_bwd, video.flow_bwd, resx, T, False, uv)
    l_prev = (mapping(xyt_b) - uv_b).norm(dim=1) * resx / (2 * uv_scale)
    return (l_prev * alpha[rows_b].squeeze()).mean() * 0.5 + (l_next * alpha[rows_f].squeeze()).mean() * 0.5


def flow_alpha_loss(video: O.Video, jif, alpha, resx, alpha_net):
    """``get_optical_flow_alpha_loss`` loss_utils.py:385-408: alpha of flow-matched points should agree."""
    T = video.T
    _, xyt_f, rows_f = O.flow_matches(jif, video.mask_fwd, video.flow_fwd, resx, T, True, alpha)
    a_f = alpha_of(alpha_net(xyt_f))
    l_next = (alpha[rows_f] - a_f).abs().mean()
    _, xyt_b, rows_b = O.flow_matches(jif, video.mask_bwd, video.flow_bwd, resx, T, False, alpha)
    a_b = alpha_of(alpha_net(xyt_b))
    l_prev = (a_b - alpha[rows_b]).abs().mean()
    return (l_next + l_prev) * 0.5


def seg_iteration_losses(video: O.Video, mask_frames: torch.Tensor, nets: Dict[str, Sequence[torch.Tensor]],
                         inds: torch.Tensor, it: int, cfg: dict = SEG_CONFIG,
                         specs: Dict[str, MlpSpec] = None, resx: int = None,
                         larger_dim: int = None) -> Dict[str, torch.Tensor]:
    """Loss terms of one trip of stage1_neural_atlas_seg.py:195-311.  ``nets`` holds the parameter lists
    'mapping1', 'mapping2', 'alpha', 'atlas'; ``mask_frames`` is the (H, W, T) bootstrapping mask.  ``resx`` and
    ``larger_dim`` override W and max(W, H) (the tests' negative controls only)."""
    specs = specs or dict(mapping1=MAPPING1_SPEC, mapping2=MAPPING2_SPEC, alpha=ALPHA_SPEC, atlas=ATLAS_SPEC)
    H, W, T = video.H, video.W, video.T
    resx = W if resx is None else resx
    larger_dim = int(np.maximum(W, H)) if larger_dim is None else larger_dim
    jif = O.pixel_table(T, H, W)[:, inds]                                    # :209
    rgb = video.frames[jif[1], jif[0], :, jif[2]].squeeze(1)                 # :211
    a_gt = mask_frames[jif[1], jif[0], jif[2]].squeeze(1).unsqueeze(-1)      # :215
    xyt = O.normalise_xyt(jif, larger_dim, T)                                # :219
    net = lambda k: (lambda x: O.mlp_forward(specs[k], nets[k], x))
    mapping1, mapping2, alpha_net, atlas = net("mapping1"), net("mapping2"), net("alpha"), net("atlas")
    uv1, uv2 = mapping1(xyt), mapping2(xyt)                                  # :225-226
    alpha = alpha_of(alpha_net(xyt))                                         # :229-232
    rgb1 = (atlas(uv1 * 0.5 + 0.5) + 1.0) * 0.5                              # :236
    rgb2 = (atlas(uv2 * 0.5 - 0.5) + 1.0) * 0.5
    rgb_out = rgb1 * alpha + rgb2 * (1.0 - alpha)                            # :240
    g = gradient_loss_seg(video, jif, mapping1, mapping2, atlas, alpha_net, rgb_out, resx)   # :243
    rgb_not = rgb1 * (1.0 - alpha)                                           # :249
    rgb_l = (torch.norm(rgb_out - rgb, dim=1) ** 2).mean()
    sparsity = (torch.norm(rgb_not, dim=1) ** 2).mean()
    s, d = cfg["uv_mapping_scale"], cfg["derivative_amount"]
    rig1 = O.rigidity_loss(jif, d, larger_dim, T, mapping1, uv1, uv_scale=s)
    rig2 = O.rigidity_loss(jif, d, larger_dim, T, mapping2, uv2, uv_scale=s)
    terms = dict(gradient=g, rgb=rgb_l, sparsity=sparsity, rigidity1=rig1, rigidity2=rig2)
    with_global = it <= cfg["stop_global_rigidity"]
    total = cfg["rigidity_coeff"] * (rig1 + rig2)
    if with_global:                                                          # :272-288
        g1 = O.rigidity_loss(jif, cfg["global_rigidity_derivative_amount_fg"], larger_dim, T, mapping1, uv1, uv_scale=s)
        g2 = O.rigidity_loss(jif, cfg["global_rigidity_derivative_amount_bg"], larger_dim, T, mapping2, uv2, uv_scale=s)
        terms.update(rigidity_global1=g1, rigidity_global2=g2)
        total = total + cfg["global_rigidity_coeff_fg"] * g1 + cfg["global_rigidity_coeff_bg"] * g2
    f1 = flow_loss_alpha(video, jif, uv1, larger_dim, mapping1, s, alpha)    # :290
    f2 = flow_loss_alpha(video, jif, uv2, larger_dim, mapping2, s, 1 - alpha)
    fa = flow_alpha_loss(video, jif, alpha, larger_dim, alpha_net)           # :300
    bce = torch.mean(-a_gt * torch.log(alpha) - (1 - a_gt) * torch.log(1 - alpha))      # :306
    boot = cfg["alpha_bootstrapping_factor"] if it <= cfg["stop_bootstrapping_iteration"] else 0
    terms.update(flow1=f1, flow2=f2, flow_alpha=fa, bootstrapping=bce)
    total = total + rgb_l * cfg["rgb_coeff"] + cfg["optical_flow_coeff"] * (f1 + f2) + bce * boot \
        + fa * cfg["alpha_flow_factor"] + sparsity * cfg["sparsity_coeff"] + g * cfg["gradient_loss_coeff"]   # :309-315
    terms["total"] = total
    return terms


def init_nets(specs: Dict[str, MlpSpec] = None):
    """Construction order of the script (:127-161): mapping1, mapping2, atlas, alpha."""
    specs = specs or dict(mapping1=MAPPING1_SPEC, mapping2=MAPPING2_SPEC, atlas=ATLAS_SPEC, alpha=ALPHA_SPEC)
    return {k: O.init_mlp(specs[k]) for k in ("mapping1", "mapping2", "atlas", "alpha")}


def make_optimizer(nets, lr: float = 1e-4):
    """:165-169 — parameter groups in the order mapping1, mapping2, alpha, atlas."""
    return torch.optim.Adam([{"params": list(nets[k])} for k in ("mapping1", "mapping2", "alpha", "atlas")], lr=lr)


def render_frame_seg(nets, f: int, H: int, W: int, T: int, specs=None, larger=None):
    """Reconstruction and alpha of frame ``f`` (evaluate.py `evaluate_model` :262-330 restricted to the RGB
    composite and alpha): (H, W, 3), (H, W).  ``larger`` overrides max(W, H) (the tests' negative controls only)."""
    specs = specs or dict(mapping1=MAPPING1_SPEC, mapping2=MAPPING2_SPEC, alpha=ALPHA_SPEC, atlas=ATLAS_SPEC)
    larger_dim = np.maximum(np.int64(W), np.int64(H)) if larger is None else np.int64(larger)
    ys, xs = torch.where(torch.ones(H, W) > 0)
    with torch.no_grad():
        xyt = torch.cat((xs.unsqueeze(1) / (larger_dim / 2) - 1, ys.unsqueeze(1) / (larger_dim / 2) - 1,
                         (f / (T / 2.0) - 1) * torch.ones(ys.shape[0], 1)), dim=1)
        a = alpha_of(O.mlp_forward(specs["alpha"], nets["alpha"], xyt))
        uv1 = O.mlp_forward(specs["mapping1"], nets["mapping1"], xyt)
        uv2 = O.mlp_forward(specs["mapping2"], nets["mapping2"], xyt)
        rgb1 = (O.mlp_forward(specs["atlas"], nets["atlas"], uv1 * 0.5 + 0.5) + 1.0) * 0.5
        rgb2 = (O.mlp_forward(specs["atlas"], nets["atlas"], uv2 * 0.5 - 0.5) + 1.0) * 0.5
        out = rgb1 * a + rgb2 * (1.0 - a)
    return out.view(H, W, 3), a.view(H, W)
