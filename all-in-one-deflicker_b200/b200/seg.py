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
import math
from typing import Dict, Optional

import numpy as np
import torch

from . import _native as N
from .atlas import DeviceVideo, FusedDp, layer_dims, make_desc, mlp_layout

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
CONSTRUCTION_ORDER = ("mapping1", "mapping2", "atlas", "alpha")   # order the script builds them (:127-161)
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


class SegTrainer:
    """Flat parameters / optimiser state of (mapping1, mapping2, alpha, atlas) + the seg step.

    Frame-sharded data parallelism: with a `process_group`, `video` holds this rank's frame block (DeviceVideo with
    t_begin / t_end and the whole-video bitmaps) and `mask` the matte of those frames (pack_mask_frames(..., t_begin,
    t_end)); every rank draws the same index batch.  A rank's trip normalises by the global batch and flow counts,
    so one SUM over the ranks of [gradients || loss vector] gives the unsharded trip (loss entries 12, 13, the flow
    counts, then read world * count).  The exchange is b200_dp_adam_step over symmetric memory (FusedDp) when
    available -- `fused_dp` True requires it, also on one rank; False or a failed set-up use NCCL all-reduce + the
    local Adam."""

    def __init__(self, video: Optional[DeviceVideo], mask: Optional[torch.Tensor], config: Optional[dict] = None,
                 precision: int = N.PREC_FP32, device="cuda", lr: float = 1e-4, resx: Optional[int] = None,
                 process_group=None, fused_dp: Optional[bool] = None):
        self.lib = N.lib()
        self.video, self.mask = video, mask
        self.cfg = dict(SEG_DEFAULTS)
        if config:
            self.cfg.update({k: v for k, v in config.items() if k in SEG_DEFAULTS})
        if float(self.cfg["global_rigidity_derivative_amount_fg"]) != float(self.cfg["global_rigidity_derivative_amount_bg"]):
            raise N.B200Error("global_rigidity_derivative_amount_fg and _bg must be equal (both 100 in the reference's config)")
        self.precision, self.device, self.lr = precision, torch.device(device), lr
        self.resx = resx if resx is not None else (video.W if video is not None else 0)
        self.descs = seg_descs(self.cfg)
        offs = (C.c_int64 * 4)()
        c0 = self._config(0)
        self.n_params = int(self.lib.b200_seg_param_floats(C.byref(c0), offs))
        if self.n_params <= 0:
            raise N.B200Error("invalid network configuration")
        self.offsets = dict(zip(NETS, [int(o) for o in offs]))
        self.layouts = {k: mlp_layout(self.descs[k]) for k in NETS}
        dev = self.device
        self.pg, self.world = process_group, 1
        if process_group is not None:
            import torch.distributed as dist
            self.world = dist.get_world_size(process_group)
        # gradients + the loss vector share one buffer so that data parallelism needs ONE exchange
        self._dp = None
        if process_group is not None and dev.type == "cuda" and fused_dp is not False and (self.world > 1 or fused_dp):
            self._dp = FusedDp.create(process_group, dev, self.n_params, N.SEG_LOSS_FLOATS, required=bool(fused_dp))
        if self._dp is None:
            self.params = torch.zeros(self.n_params, dtype=torch.float32, device=dev)
            self.grad_loss = torch.zeros(self.n_params + N.SEG_LOSS_FLOATS, dtype=torch.float32, device=dev)
        else:
            self.params, self.grad_loss = self._dp.params, self._dp.grad_loss
        self.grads = self.grad_loss[:self.n_params]
        self.losses = self.grad_loss[self.n_params:]
        self.exp_avg = torch.zeros_like(self.params)
        self.exp_avg_sq = torch.zeros_like(self.params)
        self.step_count = torch.zeros(1, dtype=torch.int64, device=dev)
        B = int(self.cfg["samples_batch"])
        self.indices = torch.zeros(B, dtype=torch.int64, device=dev)
        self._pin_inds = torch.zeros(B, dtype=torch.int64).pin_memory() if dev.type == "cuda" else None
        self._pin_loss = torch.zeros(N.SEG_LOSS_FLOATS, dtype=torch.float32).pin_memory() if dev.type == "cuda" else None
        self._ws = None
        self._render_ws = None
        self._graphs = {}

    # ------------------------------------------------------------------ parameters / state dicts
    def _views(self, flat, which):
        desc = self.descs[which]
        w, b, _ = self.layouts[which]
        base = self.offsets[which]
        out = {}
        for i, (k, n) in enumerate(layer_dims(desc)):
            out[f"hidden.{i}.weight"] = flat[base + w[i]: base + w[i] + k * n].view(n, k)
            out[f"hidden.{i}.bias"] = flat[base + b[i]: base + b[i] + n]
        return out

    def param_views(self, which):
        return self._views(self.params, which)

    def grad_views(self, which):
        return self._views(self.grads, which)

    def net_slice(self, which):
        return slice(self.offsets[which], self.offsets[which] + self.layouts[which][2])

    def init_like_reference(self):
        """nn.Linear's default init on the global CPU generator in the script's construction order
        (mapping1, mapping2, atlas, alpha), weight before bias."""
        for which in CONSTRUCTION_ORDER:
            views = self.param_views(which)
            for i, (k, n) in enumerate(layer_dims(self.descs[which])):
                bound = 1.0 / math.sqrt(k)
                views[f"hidden.{i}.weight"].copy_(torch.empty(n, k).uniform_(-bound, bound))
                views[f"hidden.{i}.bias"].copy_(torch.empty(n).uniform_(-bound, bound))

    def load_state(self, sds: Dict[str, Dict[str, torch.Tensor]]):
        for which, sd in sds.items():
            for k, v in self.param_views(which).items():
                v.copy_(sd[k].to(self.device, torch.float32))

    def state_dict(self, which):
        return {k: v.detach().clone() for k, v in self.param_views(which).items()}

    def optimizer_state_dict(self):
        """Schema of torch.optim.Adam.state_dict() for the four groups of :165-169 (what evaluate.py:223 stores).
        Collective under the fused optimiser: every rank calls it."""
        self.gather_moments()
        state, groups, idx = {}, [], 0
        step = self.step_count.detach().float().cpu().reshape(())
        for which in NETS:
            m, v = self._views(self.exp_avg, which), self._views(self.exp_avg_sq, which)
            ids = []
            for k in m:
                state[idx] = {"step": step.clone(), "exp_avg": m[k].detach().clone(), "exp_avg_sq": v[k].detach().clone()}
                ids.append(idx)
                idx += 1
            groups.append({"lr": self.lr, "betas": (0.9, 0.999), "eps": 1e-8, "weight_decay": 0, "amsgrad": False,
                           "maximize": False, "foreach": None, "capturable": False, "differentiable": False,
                           "fused": None, "params": ids})
        return {"state": state, "param_groups": groups}

    def load_optimizer_state_dict(self, sd):
        idx, step = 0, 0
        for which in NETS:
            m, v = self._views(self.exp_avg, which), self._views(self.exp_avg_sq, which)
            for k in m:
                st = sd["state"].get(idx)
                if st is not None:
                    m[k].copy_(st["exp_avg"].to(self.device))
                    v[k].copy_(st["exp_avg_sq"].to(self.device))
                    step = int(st["step"])
                idx += 1
        self.step_count.fill_(step)

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

    def adam(self, sl: Optional[slice] = None, m=None, v=None, step=None):
        sl = slice(0, self.n_params) if sl is None else sl
        N.check(self.lib.b200_adam_step(N.ptr(self.params[sl]), N.ptr(self.grads[sl]),
                                        N.ptr(self.exp_avg[sl] if m is None else m),
                                        N.ptr(self.exp_avg_sq[sl] if v is None else v), sl.stop - sl.start, self.lr,
                                        0.9, 0.999, 1e-8, 1.0, N.ptr(self.step_count if step is None else step),
                                        N.current_stream()), "b200_adam_step")

    def dp_adam(self):
        """reduce-scatter + Adam + all-gather in one kernel (b200_dp_adam_step)."""
        self._dp.adam_step(self.exp_avg, self.exp_avg_sq, self.lr, self.step_count)

    def gather_moments(self):
        """Under the fused optimiser a rank keeps the Adam moments of its slice only: assemble them (collective)."""
        if self._dp is not None:
            self._dp.gather_moments(self.exp_avg, self.exp_avg_sq)

    def all_reduce(self):
        if self.pg is not None and self.world > 1:
            import torch.distributed as dist
            dist.all_reduce(self.grad_loss, group=self.pg)      # one collective: gradients || loss vector

    def _iteration(self, it: int):
        self.loss_grad(it)
        if self._dp is not None:
            self.dp_adam()
        else:
            self.all_reduce()
            self.adam()

    def step(self, it: int, use_graph: bool = True):
        """One loop trip on the indices in self.indices (device): losses + gradients, the exchange between ranks (if
        any), then one Adam update of all four networks (same lr / betas in every group, so one sweep over the flat
        buffer).  The trip is captured once per regime (global rigidity on / off, bootstrapping on / off) in a CUDA
        graph and replayed."""
        if not use_graph or self.device.type != "cuda":
            self._iteration(it)
            return self.losses
        cfg = self._config(it)
        key = (int(cfg.with_global), float(cfg.bootstrapping_factor))
        g = self._graphs.get(key)
        if g is None:
            # eager warm-up on a side stream (builds the cached job tables), state restored afterwards; then capture
            state = (self.params, self.exp_avg, self.exp_avg_sq, self.step_count)
            snap = [t.clone() for t in state]
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                self._iteration(it)
            torch.cuda.current_stream().wait_stream(side)
            torch.cuda.synchronize()
            for t, c in zip(state, snap):
                t.copy_(c)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                self._iteration(it)
            self._graphs[key] = g
        g.replay()
        return self.losses

    def step_host(self, inds_cpu: torch.Tensor, it: int) -> np.ndarray:
        """End-to-end call with HOST buffers: pinned H2D of the index batch, one loop trip, D2H of the loss vector."""
        self._pin_inds.copy_(inds_cpu.reshape(-1))
        self.indices.copy_(self._pin_inds, non_blocking=True)
        losses = self.step(it)
        self._pin_loss.copy_(losses, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        return self._pin_loss.numpy().copy()

    def loss_dict(self, losses=None) -> Dict[str, float]:
        v = (self.losses if losses is None else torch.as_tensor(losses)).detach().float().cpu().numpy()
        return {k: float(v[i]) for i, k in enumerate(LOSS_NAMES)}

    # ------------------------------------------------------------------ pre-training
    def pretrain(self, which: str, T: int, H: int, W: int, iters: int, generator: Optional[torch.Generator] = None,
                 progress=None):
        """pre_train_mapping (unwrap_utils.py:176-198) of one of the two mapping networks: its own Adam(lr=1e-4),
        10 000 random pixels of one frame per step, index draws from the CPU generator in the reference's order."""
        desc, sl = self.descs[which], self.net_slice(which)
        n = sl.stop - sl.start
        larger = max(W, H)
        nbytes = int(self.lib.b200_mlp_pretrain_workspace_bytes(C.byref(desc), 10000))
        ws = torch.zeros(nbytes, dtype=torch.uint8, device=self.device)
        m = torch.zeros(n, dtype=torch.float32, device=self.device)
        v = torch.zeros_like(m)
        step = torch.zeros(1, dtype=torch.int64, device=self.device)
        ys_d = torch.zeros(10000, dtype=torch.int64, device=self.device)
        xs_d = torch.zeros_like(ys_d)
        loss = torch.zeros(1, dtype=torch.float32, device=self.device)
        for i in range(iters):
            for f in range(T):
                ys = torch.randint(H, (10000, 1), generator=generator)
                xs = torch.randint(W, (10000, 1), generator=generator)
                ys_d.copy_(ys.reshape(-1), non_blocking=True)
                xs_d.copy_(xs.reshape(-1), non_blocking=True)
                N.check(self.lib.b200_mlp_pretrain_loss_grad(
                    C.byref(desc), 10000, float(self.cfg["uv_mapping_scale"]), larger, T, f, N.ptr(ys_d), N.ptr(xs_d),
                    N.ptr(self.params[sl]), N.ptr(self.grads[sl]), N.ptr(loss), self.precision, N.ptr(ws), ws.numel(),
                    N.current_stream()), "b200_mlp_pretrain_loss_grad")
                self.adam(sl, m, v, step)
            if progress:
                progress(i)
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
        nbytes = int(self.lib.b200_seg_render_workspace_bytes(C.byref(cfg), chunk))
        if self._render_ws is None or self._render_ws.numel() < nbytes:
            self._render_ws = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
        ws = self._render_ws
        for p0 in range(0, H * W, chunk):
            p1 = min(H * W, p0 + chunk)
            N.check(self.lib.b200_seg_render(C.byref(cfg), N.ptr(self.params), H, W, T, f, p0, p1, N.ptr(rgb[p0 * 3:]),
                                             N.ptr(u8[p0 * 3:]) if want_u8 else None, N.ptr(alpha[p0:]), N.ptr(ws),
                                             ws.numel(), N.current_stream()), "b200_seg_render")
        out = (rgb.view(H, W, 3), alpha.view(H, W))
        return out + (u8.view(H, W, 3),) if want_u8 else out
