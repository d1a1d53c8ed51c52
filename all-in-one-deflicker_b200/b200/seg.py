"""Host side of the SEGMENTATION variant of the stage-1 loop (foreground / background mappings, alpha network, one
atlas sampled in two quadrants).  All arithmetic happens in libb200deflicker.so (csrc/seg.cu).

Mirrors, on the reference side (paths relative to the reference root):
  src/stage1_neural_atlas_seg.py:127-169   the four IMLPs + Adam over four groups
  src/stage1_neural_atlas_seg.py:195-319   one loop trip                -> SegTrainer.step
  src/models/stage_1/unwrap_utils.py:176-198  pre_train_mapping         -> SegTrainer.pretrain
  src/models/stage_1/evaluate.py:203-335   checkpoint / reconstruction  -> state dicts, render_frame
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional

import torch

from . import _native as N
from .atlas import PRETRAIN_BATCH, DeviceVideo, FlatTrainer, make_desc, mlp_layout

# hyper-parameters of src/config/config_flow_100.json that the seg loop reads
SEG_DEFAULTS = dict(
    samples_batch=10000, rgb_coeff=5000, optical_flow_coeff=500.0, gradient_loss_coeff=1000, rigidity_coeff=1.0,
    derivative_amount=1, uv_mapping_scale=0.8, include_global_rigidity_loss=True,
    global_rigidity_derivative_amount_fg=100, global_rigidity_derivative_amount_bg=100, global_rigidity_coeff_fg=5.0,
    global_rigidity_coeff_bg=50.0, stop_global_rigidity=5000, use_gradient_loss=True, alpha_bootstrapping_factor=2000.0,
    stop_bootstrapping_iteration=10000, alpha_flow_factor=4900.0, sparsity_coeff=1000.0,
    positional_encoding_num_alpha=5, number_of_channels_alpha=256, number_of_layers_alpha=8,
    use_positional_encoding_mapping1=False, number_of_positional_encoding_mapping1=4, number_of_layers_mapping1=6,
    number_of_channels_mapping1=256, use_positional_encoding_mapping2=False, number_of_positional_encoding_mapping2=2,
    number_of_layers_mapping2=4, number_of_channels_mapping2=256, number_of_channels_atlas=256, number_of_layers_atlas=8,
    positional_encoding_num_atlas=10)

NETS = ("mapping1", "mapping2", "alpha", "atlas")          # optimiser-group order (:165-169) = flat-buffer order
LOSS_NAMES = ("total", "rgb", "gradient", "sparsity", "rigidity1", "rigidity2", "rigidity_global1", "rigidity_global2",
              "flow1", "flow2", "flow_alpha", "bootstrapping", "n_fwd", "n_bwd")


def _pe_freqs(c: dict, key: str, enabled: bool = True) -> int:
    """Frequencies of an encoded network.  The reference builds a network on a 0-wide encoding when asked for 0
    frequencies; the library has no such network (pe_freqs 0 means the raw input), so that is refused."""
    if not enabled:
        return 0
    n = int(c[key])
    if n < 1:
        raise N.B200Error(f"{key} = {n}: a positionally encoded network needs at least one frequency")
    return n


def seg_descs(c: dict) -> Dict[str, N.MlpDesc]:
    """The four IMLP constructor calls of stage1_neural_atlas_seg.py:127-161."""
    return dict(
        mapping1=make_desc(3, 2, int(c["number_of_channels_mapping1"]), int(c["number_of_layers_mapping1"]),
                           _pe_freqs(c, "number_of_positional_encoding_mapping1", c["use_positional_encoding_mapping1"]), ()),
        mapping2=make_desc(3, 2, int(c["number_of_channels_mapping2"]), int(c["number_of_layers_mapping2"]),
                           _pe_freqs(c, "number_of_positional_encoding_mapping2", c["use_positional_encoding_mapping2"]), ()),
        alpha=make_desc(3, 1, int(c["number_of_channels_alpha"]), int(c["number_of_layers_alpha"]),
                        _pe_freqs(c, "positional_encoding_num_alpha"), ()),
        atlas=make_desc(2, 3, int(c["number_of_channels_atlas"]), int(c["number_of_layers_atlas"]),
                        _pe_freqs(c, "positional_encoding_num_atlas"), (4, 7)))


def pack_mask_frames(mask_frames: torch.Tensor, device, t_begin: int = 0, t_end: Optional[int] = None) -> torch.Tensor:
    """(H, W, T) bootstrapping mask of load_input_data (unwrap_utils.py:52,68-70) -> frame-major [T'][H][W] on the
    device for the resident frames [t_begin, t_end) (default: all), so that entry n of the flat buffer is pixel
    n + t_begin*H*W of the index table.  A frame shard's trainer takes the matte of its own frames only."""
    return mask_frames[:, :, t_begin:t_end].permute(2, 0, 1).contiguous().to(device=device, dtype=torch.float32)


class SegTrainer(FlatTrainer):
    """Flat parameters / optimiser state of (mapping1, mapping2, alpha, atlas) + the seg step.

    Frame-sharded data parallelism: with a `process_group`, `video` holds this rank's frame block (DeviceVideo with
    t_begin / t_end and the whole-video bitmaps) and `mask` the matte of those frames (pack_mask_frames(..., t_begin,
    t_end)); every rank draws the same index batch.  A rank's trip normalises by the global batch and flow counts,
    so one SUM over the ranks of [gradients || loss vector] gives the unsharded trip (loss entries 12, 13, the flow
    counts, then read world * count).  FlatTrainer describes the exchange and `fused_dp`."""

    NETS = NETS
    CONSTRUCTION_ORDER = ("mapping1", "mapping2", "atlas", "alpha")   # order the script builds them (:127-161)

    def __init__(self, video: Optional[DeviceVideo], mask: Optional[torch.Tensor], config: Optional[dict] = None,
                 precision: int = N.PREC_FP32, device="cuda", lr: float = 1e-4, resx: Optional[int] = None,
                 process_group=None, fused_dp: Optional[bool] = None):
        super().__init__(video, precision, device, lr, process_group, resx)
        self.mask = mask
        self.cfg = dict(SEG_DEFAULTS)
        if config:
            self.cfg.update({k: v for k, v in config.items() if k in SEG_DEFAULTS})
        if float(self.cfg["global_rigidity_derivative_amount_fg"]) != float(self.cfg["global_rigidity_derivative_amount_bg"]):
            raise N.B200Error("global_rigidity_derivative_amount_fg and _bg must be equal (both 100 in the reference's config)")
        self.descs = seg_descs(self.cfg)
        offs = (C.c_int64 * 4)()
        c0 = self._config(0)
        self.n_params = int(self.lib.b200_seg_param_floats(C.byref(c0), offs))
        if self.n_params <= 0:
            raise N.B200Error("invalid network configuration")
        self.offsets = dict(zip(NETS, [int(o) for o in offs]))
        self.layouts = {k: mlp_layout(self.descs[k]) for k in NETS}
        self._allocate(N.SEG_LOSS_FLOATS, fused_dp)

    # ------------------------------------------------------------------ native calls
    def _config(self, it: int) -> N.SegConfig:
        c = self.cfg
        with_global = bool(c["include_global_rigidity_loss"]) and it <= int(c["stop_global_rigidity"])   # :272
        boot = float(c["alpha_bootstrapping_factor"]) if it <= int(c["stop_bootstrapping_iteration"]) else 0.0   # :198
        d = seg_descs(c)
        return N.SegConfig(int(c["samples_batch"]), 1 if with_global else 0, self.precision, int(self.resx),
                           float(c["uv_mapping_scale"]), float(c["derivative_amount"]),
                           float(c["global_rigidity_derivative_amount_fg"]), float(c["rgb_coeff"]),
                           float(c["gradient_loss_coeff"]) if c["use_gradient_loss"] else 0.0, float(c["rigidity_coeff"]),
                           float(c["global_rigidity_coeff_fg"]), float(c["global_rigidity_coeff_bg"]),
                           float(c["optical_flow_coeff"]), float(c["alpha_flow_factor"]), float(c["sparsity_coeff"]), boot,
                           d["mapping1"], d["mapping2"], d["alpha"], d["atlas"])

    def _workspace(self):
        if self._ws is None:
            c = self._config(0)
            n = int(self.lib.b200_seg_workspace_bytes(C.byref(c)))
            if n <= 0:
                raise N.B200Error("b200_seg_workspace_bytes: " + N.last_error())
            self._ws = torch.zeros(n, dtype=torch.uint8, device=self.device)
        return self._ws

    def loss_grad(self, it: int):
        cfg, ws = self._config(it), self._workspace()
        N.check(self.lib.b200_seg_loss_grad(C.byref(cfg), C.byref(self.video.struct), N.ptr(self.mask), N.ptr(self.indices),
                                            N.ptr(self.params), N.ptr(self.grads), N.ptr(self.losses), N.ptr(ws),
                                            ws.numel(), N.current_stream()), "b200_seg_loss_grad")

    def _trip(self, it: int):
        self.loss_grad(it)

    def _regime(self, it: int):
        """Global rigidity on / off and bootstrapping on / off."""
        cfg = self._config(it)
        return int(cfg.with_global), float(cfg.bootstrapping_factor)

    def loss_dict(self, losses=None) -> Dict[str, float]:
        v = (self.losses if losses is None else torch.as_tensor(losses)).detach().float().cpu().numpy()
        return {k: float(v[i]) for i, k in enumerate(LOSS_NAMES)}

    # ------------------------------------------------------------------ pre-training
    def pretrain(self, which: str, T: int, H: int, W: int, iters: int, generator: Optional[torch.Generator] = None,
                 progress=None):
        """pre_train_mapping of one of the two mapping networks (FlatTrainer._pretrain).  Returns the device loss of
        the last step."""
        desc, sl = self.descs[which], self.net_slice(which)
        larger = max(W, H)
        nbytes = int(self.lib.b200_mlp_pretrain_workspace_bytes(C.byref(desc), PRETRAIN_BATCH))
        ws = torch.zeros(nbytes, dtype=torch.uint8, device=self.device)
        loss = torch.zeros(1, dtype=torch.float32, device=self.device)

        def loss_grad(f, ys, xs):
            N.check(self.lib.b200_mlp_pretrain_loss_grad(
                C.byref(desc), PRETRAIN_BATCH, float(self.cfg["uv_mapping_scale"]), larger, T, f, N.ptr(ys), N.ptr(xs),
                N.ptr(self.params[sl]), N.ptr(self.grads[sl]), N.ptr(loss), self.precision, N.ptr(ws), ws.numel(),
                N.current_stream()), "b200_mlp_pretrain_loss_grad")
        self._pretrain(sl, T, H, W, iters, generator, progress, loss_grad)
        return loss

    # ------------------------------------------------------------------ reconstruction
    def render_frame(self, f: int, H: int, W: int, T: int, chunk: int = 65536, want_u8: bool = False):
        """Composite reconstruction and alpha of frame f (evaluate.py:293-335): (H, W, 3) fp32, (H, W) fp32
        [and uint8 by truncation]."""
        chunk = min(chunk, H * W)
        cfg = self._config(0)
        rgb = torch.empty(H * W * 3, dtype=torch.float32, device=self.device)
        alpha = torch.empty(H * W, dtype=torch.float32, device=self.device)
        u8 = torch.empty(H * W * 3, dtype=torch.uint8, device=self.device) if want_u8 else None
        ws = self._scratch_buffer("render", int(self.lib.b200_seg_render_workspace_bytes(C.byref(cfg), chunk)))
        for p0 in range(0, H * W, chunk):
            p1 = min(H * W, p0 + chunk)
            N.check(self.lib.b200_seg_render(C.byref(cfg), N.ptr(self.params), H, W, T, f, p0, p1, N.ptr(rgb[p0 * 3:]),
                                             N.ptr(u8[p0 * 3:]) if want_u8 else None, N.ptr(alpha[p0:]), N.ptr(ws),
                                             ws.numel(), N.current_stream()), "b200_seg_render")
        out = (rgb.view(H, W, 3), alpha.view(H, W))
        return out + (u8.view(H, W, 3),) if want_u8 else out
