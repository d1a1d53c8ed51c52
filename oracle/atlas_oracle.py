"""CPU restatement (oracle) of the reference's stage-1 neural-atlas arithmetic.

TEST INFRASTRUCTURE ONLY.  Nothing under ``oracle/`` is part of the product: only
``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s cpu_baseline / ``--impl
reference`` legs may import it, and there only as the checker / CPU baseline.

Parity pinning: the reference ships no tests and no golden vectors (SURVEY.md §4), so
this restatement is pinned against the reference's *own modules executed in the build
container* (``tests/golden/make_golden.py`` imports ``/root/reference`` and asserts
bit-equality with the functions below, then freezes small input/output fixtures under
``tests/golden/``).  ``tests/test_oracle_golden.py`` replays those fixtures.

Every function cites the reference lines it restates (paths relative to the reference
root).  The arithmetic is written with the same torch primitives in the same order as
the reference wherever fp32 rounding depends on it (division of int64 tensors by numpy
float scalars, ``norm(dim=1) ** 2``, ...), but the structure is functional: networks
are plain lists of (weight, bias) tensors and the video is a small dataclass.
"""
from __future__ import annotations

import dataclasses
import math
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.nn.functional as F


# ----------------------------------------------------------------------------------------
# IMLP  (src/models/stage_1/implicit_neural_networks.py:9-81)
# ----------------------------------------------------------------------------------------
@dataclasses.dataclass(frozen=True)
class MlpSpec:
    """Shape of one IMLP, ctor arguments of implicit_neural_networks.py:16-25."""
    input_dim: int
    output_dim: int
    hidden_dim: int = 256
    use_positional: bool = True
    positional_dim: int = 10
    skip_layers: Tuple[int, ...] = (4, 6)
    num_layers: int = 8
    use_tanh: bool = True

    @property
    def enc_dim(self) -> int:  # implicit_neural_networks.py:32-36
        return 2 * self.input_dim * self.positional_dim if self.use_positional else self.input_dim

    def layer_dims(self) -> List[Tuple[int, int]]:
        """(fan_in, fan_out) per Linear, implicit_neural_networks.py:39-52."""
        dims = []
        for i in range(self.num_layers):
            if i == 0:
                k = self.enc_dim
            elif i in self.skip_layers:
                k = self.hidden_dim + self.enc_dim
            else:
                k = self.hidden_dim
            n = self.output_dim if i == self.num_layers - 1 else self.hidden_dim
            dims.append((k, n))
        return dims

    def num_params(self) -> int:
        return sum(k * n + n for k, n in self.layer_dims())


# the two networks the non-segmentation script builds (src/stage1_neural_atlas.py:112-128
# with src/config/config_flow_100.json values)
MAPPING_SPEC = MlpSpec(3, 2, 256, False, 4, (), 6)
ATLAS_SPEC = MlpSpec(2, 3, 256, True, 10, (4, 7), 8)


def pe_frequencies(spec: MlpSpec) -> torch.Tensor:
    """``b`` of implicit_neural_networks.py:34 — float64 products rounded to fp32."""
    return torch.tensor([(2 ** j) * np.pi for j in range(spec.positional_dim)])


def positional_encoding(x: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """implicit_neural_networks.py:9-13.  Row layout: for each frequency k the block
    [sin(x_0 b_k) .. sin(x_{d-1} b_k), cos(x_0 b_k) .. cos(x_{d-1} b_k)]."""
    proj = x[:, :, None] * b.to(x.dtype)[None, None, :]          # (rows, d, F); one fp mult each (b is fp32-valued)
    sc = torch.cat((torch.sin(proj), torch.cos(proj)), dim=1)     # (rows, 2d, F)
    return sc.transpose(2, 1).reshape(x.shape[0], -1)             # (rows, F*2d)


def init_mlp(spec: MlpSpec, generator: Optional[torch.Generator] = None) -> List[torch.Tensor]:
    """Parameters [W0, b0, W1, b1, ...] drawn exactly like ``nn.Linear`` does
    (implicit_neural_networks.py:48-52 → torch.nn.Linear.reset_parameters:
    kaiming_uniform(a=sqrt 5) on the weight = U(-1/sqrt(k), 1/sqrt(k)), same bound for
    the bias), consuming the RNG in layer order, weight before bias."""
    params = []
    for k, n in spec.layer_dims():
        bound = 1.0 / math.sqrt(k)
        w = torch.empty(n, k).uniform_(-bound, bound, generator=generator)
        bb = torch.empty(n).uniform_(-bound, bound, generator=generator)
        params += [w, bb]
    return params


def mlp_forward(spec: MlpSpec, params: Sequence[torch.Tensor], x: torch.Tensor) -> torch.Tensor:
    """implicit_neural_networks.py:62-81.  (Inputs are cast to the parameter dtype: a no-op for the
    fp32 reference arithmetic, and what lets the tests build a float64 "truth" with float64 params.)"""
    x = x.to(params[0].dtype)
    if spec.use_positional:
        x = positional_encoding(x, pe_frequencies(spec).to(x.device))
    skip_in = x.detach().clone()                                   # :69 — detached skip input
    for i in range(spec.num_layers):
        if i > 0:
            x = F.relu(x)
        if i in spec.skip_layers:
            x = torch.cat((x, skip_in), 1)
        x = F.linear(x, params[2 * i], params[2 * i + 1])
    if spec.use_tanh:
        x = torch.tanh(x)
    return x


def state_dict_of(params: Sequence[torch.Tensor]) -> Dict[str, torch.Tensor]:
    """Keys of ``IMLP.state_dict()``: hidden.{i}.weight / hidden.{i}.bias."""
    out = {}
    for i in range(len(params) // 2):
        out[f"hidden.{i}.weight"] = params[2 * i]
        out[f"hidden.{i}.bias"] = params[2 * i + 1]
    return out


# ----------------------------------------------------------------------------------------
# video container + index table  (src/models/stage_1/unwrap_utils.py:105-173)
# ----------------------------------------------------------------------------------------
@dataclasses.dataclass
class Video:
    """The eight CPU tensors ``load_input_data_single`` returns, reference layouts
    (unwrap_utils.py:112-122): T innermost."""
    frames: torch.Tensor        # (H, W, 3, T) fp32 in [0,1]
    frames_dx: torch.Tensor     # (H, W, 3, T) forward difference along x, 0 in last column
    frames_dy: torch.Tensor     # (H, W, 3, T) forward difference along y, 0 in last row
    flow_fwd: torch.Tensor      # (H, W, 2, T, 1) flow t -> t+1 in pixels
    flow_bwd: torch.Tensor      # (H, W, 2, T, 1) flow t -> t-1 in pixels
    mask_fwd: torch.Tensor      # (H, W, T, 1) 0/1 fp32
    mask_bwd: torch.Tensor      # (H, W, T, 1) 0/1 fp32

    @property
    def H(self): return self.frames.shape[0]
    @property
    def W(self): return self.frames.shape[1]
    @property
    def T(self): return self.frames.shape[3]


def image_differences(frames: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """unwrap_utils.py:132-133."""
    dx = torch.zeros_like(frames)
    dy = torch.zeros_like(frames)
    dy[:-1] = frames[1:] - frames[:-1]
    dx[:, :-1] = frames[:, 1:] - frames[:, :-1]
    return dx, dy


def pixel_table(T: int, H: int, W: int) -> torch.Tensor:
    """``get_tuples`` (unwrap_utils.py:166-173): (3, T*H*W) int64 rows [x; y; t], pixels of a
    frame in row-major (y, x) order, frames concatenated — i.e. n -> (n % W, (n // W) % H,
    n // (H*W)).  (Every pixel passes the ``> -1`` test for image data.)"""
    n = torch.arange(T * H * W, dtype=torch.int64)
    return torch.stack((n % W, (n // W) % H, n // (H * W)))


# ----------------------------------------------------------------------------------------
# coordinate normalisation (int64 tensor / numpy-float64 scalar -> fp32, SURVEY §8c)
# ----------------------------------------------------------------------------------------
def _half(v) -> np.float64:
    return np.float64(v) / 2


def normalise_xyt(jif: torch.Tensor, larger_dim: int, T: int) -> torch.Tensor:
    """src/stage1_neural_atlas.py:168-171.  ``jif`` is (3, B, 1) int64."""
    return torch.cat((jif[0] / _half(larger_dim) - 1,
                      jif[1] / _half(larger_dim) - 1,
                      jif[2] / (T / 2.0) - 1), dim=1)


# ----------------------------------------------------------------------------------------
# losses  (src/models/stage_1/loss_utils.py)
# ----------------------------------------------------------------------------------------
def gradient_loss(video: Video, jif, mapping, atlas, rgb_out, resx: int):
    """``get_gradient_loss_single`` loss_utils.py:134-170 (coordinates are normalised by
    the ``resx`` argument the caller passes, src/stage1_neural_atlas.py:186-188)."""
    T = video.T
    xp = torch.cat(((jif[0] + 1) / _half(resx) - 1, jif[1] / _half(resx) - 1,
                    jif[2] / (T / 2.0) - 1), dim=1)
    yp = torch.cat((jif[0] / _half(resx) - 1, (jif[1] + 1) / _half(resx) - 1,
                    jif[2] / (T / 2.0) - 1), dim=1)
    dx_gt = video.frames_dx[jif[1], jif[0], :, jif[2]].squeeze(1).to(rgb_out.device)   # loss_utils.py:148-151
    dy_gt = video.frames_dy[jif[1], jif[0], :, jif[2]].squeeze(1).to(rgb_out.device)
    uv_yp = mapping(yp)
    uv_xp = mapping(xp)
    rgb_yp = (atlas(uv_yp * 0.5 + 0.5) + 1.0) * 0.5
    rgb_xp = (atlas(uv_xp * 0.5 + 0.5) + 1.0) * 0.5
    dx_out = rgb_xp - rgb_out
    dy_out = rgb_yp - rgb_out
    return torch.mean((dx_gt - dx_out).norm(dim=1) ** 2 + (dy_gt - dy_out).norm(dim=1) ** 2)


def rigidity_loss(jif, d: int, resx, T: int, mapping, uv, uv_scale: float = 1.0,
                  per_sample: bool = False):
    """``get_rigidity_loss`` loss_utils.py:227-278."""
    ys = torch.cat((jif[1] - d, jif[1])) / _half(resx) - 1
    xs = torch.cat((jif[0], jif[0] - d)) / _half(resx) - 1
    ts = torch.cat((jif[2], jif[2])) / (T / 2.0) - 1
    uv_p = mapping(torch.cat((xs, ys, ts), dim=1))
    u_p = uv_p[:, 0].view(2, -1)
    v_p = uv_p[:, 1].view(2, -1)
    du = uv[:, 0].unsqueeze(0) - u_p          # [0]: d/dy   [1]: d/dx
    dv = uv[:, 1].unsqueeze(0) - v_p
    du_dx = du[1] * resx / 2
    du_dy = du[0] * resx / 2
    dv_dy = dv[0] * resx / 2
    dv_dx = dv[1] * resx / 2
    J = torch.stack((torch.stack((du_dx, du_dy), dim=1), torch.stack((dv_dx, dv_dy), dim=1)), dim=1)
    J = J / uv_scale
    J = J / d
    JtJ = torch.matmul(J.transpose(1, 2), J)
    a = JtJ[:, 0, 0] + 0.001
    b = JtJ[:, 0, 1]
    c = JtJ[:, 1, 0]
    dd = JtJ[:, 1, 1] + 0.001
    adj = torch.stack((torch.stack((dd, -b), dim=1), torch.stack((-c, a), dim=1)), dim=1)
    inv = adj / ((a * dd - b * c).unsqueeze(-1).unsqueeze(-1))
    out = (JtJ ** 2).sum(1).sum(1).sqrt() + (inv ** 2).sum(1).sum(1).sqrt()
    return out if per_sample else out.mean()


def flow_matches(jif, mask, flow, resx, T: int, forward: bool, uv):
    """``get_corresponding_flow_matches`` loss_utils.py:326-356 (single flow level)."""
    sel = torch.where(mask[jif[1].squeeze(), jif[0].squeeze(), jif[2].squeeze(), :])
    step = 2 ** sel[1]
    rows = sel[0]
    j = jif[:, rows, 0]
    fl = flow[j[1], j[0], :, j[2], sel[1]]
    tt = j[2] + step if forward else j[2] - step
    m = torch.stack((j[0] + fl[:, 0], j[1] + fl[:, 1], tt))
    xyt = torch.stack((m[0] / _half(resx) - 1, m[1] / _half(resx) - 1, m[2] / (T / 2) - 1)).T
    return uv[rows], xyt, rows


def flow_loss(video: Video, jif, uv, resx, mapping, uv_scale: float):
    """``get_optical_flow_loss`` loss_utils.py:299-322 with alpha == 1
    (src/stage1_neural_atlas.py:177,215-218).  Empty relevant set -> NaN, as there."""
    T = video.T
    uv_f, xyt_f, _ = flow_matches(jif, video.mask_fwd, video.flow_fwd, resx, T, True, uv)
    l_next = (mapping(xyt_f) - uv_f).norm(dim=1) * resx / (2 * uv_scale)
    uv_b, xyt_b, _ = flow_matches(jif, video.mask_bwd, video.flow_bwd, resx, T, False, uv)
    l_prev = (mapping(xyt_b) - uv_b).norm(dim=1) * resx / (2 * uv_scale)
    return l_prev.mean() * 0.5 + l_next.mean() * 0.5


def flow_loss_all(video: Video, jif, uv, resx, T: int, mapping, uv_scale: float):
    """``get_optical_flow_loss_all`` loss_utils.py:283-295 (+ ``get_corresponding_flow_matches_all`` :360-382) with
    alpha == 1: forward flow error of EVERY sample, zero where the flow is invalid."""
    fl = video.flow_fwd[jif[1], jif[0], :, jif[2], 0].squeeze()
    ok = video.mask_fwd[jif[1], jif[0], jif[2], 0].squeeze()
    m = torch.stack((jif[0].squeeze() + fl[:, 0], jif[1].squeeze() + fl[:, 1], jif[2].squeeze() + 1))
    xyt = torch.stack((m[0] / _half(resx) - 1, m[1] / _half(resx) - 1, m[2] / (T / 2) - 1)).T
    err = (mapping(xyt) - uv).norm(dim=1)
    err[(ok > 0) == False] = 0                      # noqa: E712  (the reference's comparison, loss_utils.py:292)
    return err * resx / (2 * uv_scale)


def eval_maps(video: Video, map_params, f: int, d: int = 1, uv_scale: float = 0.8, larger=None):
    """Per-pixel maps of frame ``f`` as the reference's evaluation computes them (evaluate.py:640-700): uv (H, W, 2),
    rigidity loss (H, W), forward flow error (H, W; zero for the last frame).  ``larger`` overrides max(W, H) (the
    tests' negative controls only)."""
    H, W, T = video.H, video.W, video.T
    larger = np.maximum(np.int64(W), np.int64(H)) if larger is None else np.int64(larger)
    ys, xs = torch.where(torch.ones(H, W) > 0)
    mapping = lambda x: mlp_forward(MAPPING_SPEC, map_params, x)
    with torch.no_grad():
        xyt = torch.cat((xs.unsqueeze(1) / (larger / 2) - 1, ys.unsqueeze(1) / (larger / 2) - 1,
                         (f / (T / 2.0) - 1) * torch.ones(ys.shape[0], 1)), dim=1)
        uv = mapping(xyt)
        jif = torch.cat((xs.unsqueeze(-1), ys.unsqueeze(-1), torch.ones_like(ys.unsqueeze(-1)) * f), dim=1).T.unsqueeze(-1)
        rig = rigidity_loss(jif, d, larger, T, mapping, uv, uv_scale=uv_scale, per_sample=True)
        flow = flow_loss_all(video, jif, uv, larger, T, mapping, uv_scale) if f < T - 1 else torch.zeros(ys.shape[0])
    return uv.view(H, W, 2), rig.view(H, W), flow.view(H, W)


# ----------------------------------------------------------------------------------------
# one iteration of the hot loop  (src/stage1_neural_atlas.py:151-231)
# ----------------------------------------------------------------------------------------
DEFAULT_CONFIG = dict(rgb_coeff=5000, optical_flow_coeff=500.0, gradient_loss_coeff=1000,
                      rigidity_coeff=1.0, derivative_amount=1, uv_mapping_scale=0.8,
                      global_rigidity_derivative_amount_fg=100, global_rigidity_coeff_fg=5.0,
                      stop_global_rigidity=5000, samples_batch=10000, iters_num=10001,
                      pretrain_iter_number=100)


def iteration_losses(video: Video, map_params, atlas_params, inds: torch.Tensor, it: int,
                     cfg: dict = DEFAULT_CONFIG, device: str = "cpu", resx: Optional[int] = None,
                     larger_dim: Optional[int] = None) -> Dict[str, torch.Tensor]:
    """Loss terms of one loop trip for sample indices ``inds`` ((B,1) int64 into the pixel
    table).  Returns the individual terms and the weighted ``total`` (with grad).  ``resx`` and
    ``larger_dim`` override W and max(W, H) (the tests' negative controls only)."""
    H, W, T = video.H, video.W, video.T
    resx = W if resx is None else resx
    larger_dim = int(np.maximum(W, H)) if larger_dim is None else larger_dim
    table = pixel_table(T, H, W)
    jif = table[:, inds]                                            # (3, B, 1)  :162
    rgb = video.frames[jif[1], jif[0], :, jif[2]].squeeze(1).to(device)     # :164
    xyt = normalise_xyt(jif, larger_dim, T).to(device)             # :168
    mapping = lambda x: mlp_forward(MAPPING_SPEC, map_params, x.to(device))
    atlas = lambda x: mlp_forward(ATLAS_SPEC, atlas_params, x)
    uv = mapping(xyt)                                              # :174
    rgb_out = (atlas(uv * 0.5 + 0.5) + 1.0) * 0.5                  # :181
    g = gradient_loss(video_to(video, "cpu"), jif, mapping, atlas, rgb_out, resx)   # :186
    rgb_l = (torch.norm(rgb_out - rgb, dim=1) ** 2).mean()         # :194
    rig = rigidity_loss(jif, cfg["derivative_amount"], larger_dim, T, mapping, uv,
                        uv_scale=cfg["uv_mapping_scale"])          # :196
    with_global = it <= cfg["stop_global_rigidity"]
    terms = dict(gradient=g, rgb=rgb_l, rigidity=rig)
    total = cfg["rigidity_coeff"] * rig
    if with_global:                                                # :205
        rig_g = rigidity_loss(jif, cfg["global_rigidity_derivative_amount_fg"], larger_dim, T,
                              mapping, uv, uv_scale=cfg["uv_mapping_scale"])
        terms["rigidity_global"] = rig_g
        total = total + cfg["global_rigidity_coeff_fg"] * rig_g
    fl = flow_loss(video, jif, uv, larger_dim, mapping, cfg["uv_mapping_scale"])   # :215
    terms["flow"] = fl
    total = total + rgb_l * cfg["rgb_coeff"] + cfg["optical_flow_coeff"] * fl \
        + g * cfg["gradient_loss_coeff"]                           # :220-227
    terms["total"] = total
    return terms


def video_to(video: Video, device) -> Video:
    return video  # the reference keeps all video tensors on the CPU (SURVEY §3.2 step 2)


def pretrain_losses(map_params, frame: int, ys: torch.Tensor, xs: torch.Tensor, T: int,
                    larger_dim: int, uv_scale: float, device: str = "cpu") -> torch.Tensor:
    """Loss of one ``pre_train_mapping`` step (unwrap_utils.py:182-195) for already drawn
    integer rows ``ys`` / columns ``xs`` ((B,1) int64)."""
    i_s = ys / _half(larger_dim) - 1
    j_s = xs / _half(larger_dim) - 1
    xyt = torch.cat((j_s, i_s, (frame / (T / 2.0) - 1) * torch.ones_like(i_s)), dim=1).to(device)
    uv = mlp_forward(MAPPING_SPEC, map_params, xyt)
    return (xyt[:, :2] * uv_scale - uv).norm(dim=1).mean()


def make_optimizer(map_params, atlas_params, lr: float = 1e-4):
    """src/stage1_neural_atlas.py:132-134."""
    return torch.optim.Adam([{"params": list(map_params)}, {"params": list(atlas_params)}], lr=lr)


def train_iteration(video, map_params, atlas_params, opt, inds, it, cfg=DEFAULT_CONFIG,
                    device: str = "cpu"):
    """zero_grad / backward / step of src/stage1_neural_atlas.py:229-231."""
    terms = iteration_losses(video, map_params, atlas_params, inds, it, cfg, device)
    opt.zero_grad()
    terms["total"].backward()
    opt.step()
    return {k: float(v.detach()) for k, v in terms.items()}


# ----------------------------------------------------------------------------------------
# render + PSNR  (src/models/stage_1/evaluate.py:640-708, 733, 740-743)
# ----------------------------------------------------------------------------------------
def render_frame(map_params, atlas_params, f: int, H: int, W: int, T: int,
                 chunk: int = 100000, device: str = "cpu", larger=None) -> torch.Tensor:
    """RGB reconstruction of frame ``f`` as (H, W, 3) fp32; evaluate.py:644-666 (pixels of the
    frame in row-major order, split with np.array_split into <=100k chunks).  ``larger`` overrides
    max(W, H) (the tests' negative controls only)."""
    larger_dim = np.maximum(np.int64(W), np.int64(H)) if larger is None else np.int64(larger)
    ys, xs = torch.where(torch.ones(H, W) > 0)
    parts = int(np.ceil(ys.shape[0] / chunk))
    out = torch.zeros(H, W, 3)
    with torch.no_grad():
        for yy, xx in zip(np.array_split(ys.numpy(), parts), np.array_split(xs.numpy(), parts)):
            ry = torch.from_numpy(yy).unsqueeze(1) / (larger_dim / 2) - 1
            rx = torch.from_numpy(xx).unsqueeze(1) / (larger_dim / 2) - 1
            xyt = torch.cat((rx, ry, (f / (T / 2.0) - 1) * torch.ones_like(ry)), dim=1).to(device)
            uv = mlp_forward(MAPPING_SPEC, map_params, xyt)
            rgb = (mlp_forward(ATLAS_SPEC, atlas_params, uv * 0.5 + 0.5) + 1) * 0.5
            out[yy, xx] = rgb.cpu()
    return out


def to_uint8(img: torch.Tensor) -> np.ndarray:
    """evaluate.py:733 — ``(x * 255).astype(np.uint8)`` on a float64 array: truncation."""
    return (img.double().numpy() * 255).astype(np.uint8)


def psnr(a: torch.Tensor, b: torch.Tensor) -> float:
    """skimage.metrics.peak_signal_noise_ratio(data_range=1) as used at evaluate.py:740-743:
    10 log10(1 / mean((a-b)^2)) in float64."""
    err = np.mean((a.double().numpy() - b.double().numpy()) ** 2)
    return float(10 * np.log10(1.0 / err))
