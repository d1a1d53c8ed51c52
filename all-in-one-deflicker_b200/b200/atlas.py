"""Host side of the fused stage-1 atlas loop: device video, flat parameters, CUDA-graph replay,
frame-sharded data parallelism.  All arithmetic happens in libb200deflicker.so.

Mirrors, on the reference side (paths relative to the reference root):
  src/stage1_neural_atlas.py:106-134   data + the two IMLPs + Adam
  src/stage1_neural_atlas.py:151-231   one loop trip            -> AtlasTrainer.step
  src/models/stage_1/unwrap_utils.py:176-198  pre_train_mapping -> AtlasTrainer.pretrain
  src/models/stage_1/evaluate.py:616-666,733-743  checkpoint / render / PSNR
"""
from __future__ import annotations

import ctypes as C
import math
from typing import Dict, Optional

import numpy as np
import torch

from . import _native as N

# hyper-parameters of src/config/config_flow_100.json that the loop reads
DEFAULTS = dict(samples_batch=10000, rgb_coeff=5000, optical_flow_coeff=500.0, gradient_loss_coeff=1000,
                rigidity_coeff=1.0, derivative_amount=1, uv_mapping_scale=0.8,
                include_global_rigidity_loss=True, global_rigidity_derivative_amount_fg=100,
                global_rigidity_coeff_fg=5.0, stop_global_rigidity=5000, use_gradient_loss=True)
# pre_train_mapping draws 10000 pixels per step, whatever samples_batch is (unwrap_utils.py:183)
PRETRAIN_BATCH = 10000

MAPPING_DESC = dict(input_dim=3, output_dim=2, hidden_dim=256, num_layers=6, pe_freqs=0, skip_layers=())
ATLAS_DESC = dict(input_dim=2, output_dim=3, hidden_dim=256, num_layers=8, pe_freqs=10, skip_layers=(4, 7))


def make_desc(input_dim, output_dim, hidden_dim, num_layers, pe_freqs, skip_layers, use_tanh=True) -> N.MlpDesc:
    mask = 0
    for s in skip_layers:
        mask |= 1 << int(s)
    return N.MlpDesc(input_dim, output_dim, hidden_dim, num_layers, pe_freqs, mask, 1 if use_tanh else 0, 0)


def mlp_layout(desc: N.MlpDesc):
    w = (C.c_int64 * N.MAX_LAYERS)()
    b = (C.c_int64 * N.MAX_LAYERS)()
    total = N.lib().b200_mlp_layout(C.byref(desc), w, b)
    if total < 0:
        raise N.B200Error("invalid IMLP descriptor: " + N.lib().b200_last_error().decode())
    return list(w[:desc.num_layers]), list(b[:desc.num_layers]), int(total)


def layer_dims(desc: N.MlpDesc):
    enc = 2 * desc.input_dim * desc.pe_freqs if desc.pe_freqs > 0 else desc.input_dim
    dims = []
    for i in range(desc.num_layers):
        k = enc if i == 0 else (desc.hidden_dim + enc if (desc.skip_mask >> i) & 1 else desc.hidden_dim)
        n = desc.output_dim if i == desc.num_layers - 1 else desc.hidden_dim
        dims.append((k, n))
    return dims


class DeviceVideo:
    """Frame-major pixel records + whole-video validity bitmaps in HBM (B200Video)."""

    def __init__(self, H, W, T, t_begin, t_end, records, bits_f, bits_b):
        self.H, self.W, self.T, self.t_begin, self.t_end = H, W, T, t_begin, t_end
        self.records, self.bits_f, self.bits_b = records, bits_f, bits_b
        self.struct = N.Video(records.data_ptr(), bits_f.data_ptr(), bits_b.data_ptr(), H, W, T, t_begin, t_end, 0)

    @property
    def num_pixels(self):
        return self.H * self.W * self.T

    def frame_rgb(self, f: int) -> torch.Tensor:
        """The fp32 frame f as held in channels 0..2 of its resident records: an (H, W, 3) device tensor (a copy)."""
        if not self.t_begin <= f < self.t_end:
            raise N.B200Error(f"frame {f} is not resident (frames [{self.t_begin}, {self.t_end}))")
        HW = self.H * self.W
        rec = self.records[(f - self.t_begin) * HW * N.RECORD_FLOATS:(f - self.t_begin + 1) * HW * N.RECORD_FLOATS]
        return rec.view(HW, N.RECORD_FLOATS)[:, :3].reshape(self.H, self.W, 3)

    def mask_fwd_host(self) -> torch.Tensor:
        """The forward consistency masks as the reference's (H, W, T, 1) fp32 CPU tensor, unpacked from the bitmap."""
        n = self.num_pixels
        words = self.bits_f.cpu().numpy().view(np.uint32)
        bits = np.unpackbits(words.view(np.uint8), bitorder="little")[:n]
        return torch.from_numpy(bits.reshape(self.T, self.H, self.W).astype(np.float32)).permute(1, 2, 0).unsqueeze(-1).contiguous()

    @classmethod
    def from_reference_layout(cls, data: Dict[str, torch.Tensor], device, t_begin: int = 0,
                              t_end: Optional[int] = None, frame_chunk: int = 16) -> "DeviceVideo":
        """`data`: CPU tensors in the layouts of load_input_data_single (unwrap_utils.py:112-122).
        Uploaded and repacked `frame_chunk` frames at a time so the staging copy stays small."""
        fr = data["frames"]
        H, W, _, T = fr.shape
        t_end = T if t_end is None else t_end
        lib = N.lib()
        n_local = H * W * (t_end - t_begin)
        records = torch.empty(max(n_local, 1) * N.RECORD_FLOATS, dtype=torch.float32, device=device)
        words = (H * W * T + 31) // 32
        bits_f = torch.zeros(words, dtype=torch.int32, device=device)
        bits_b = torch.zeros(words, dtype=torch.int32, device=device)
        # masks for the whole video (small: H*W*T floats), frames/flows only for the resident range
        mf = data["mask_fwd"].to(device, non_blocking=False).contiguous()
        mb = data["mask_bwd"].to(device).contiguous()
        st = N.current_stream()
        keys = ("frames", "frames_dx", "frames_dy", "flow_fwd", "flow_bwd")
        t0 = t_begin
        first = True
        while first or t0 < t_end:
            t1 = min(t_end, t0 + frame_chunk)
            # a chunk [t0,t1) is staged as its own little "video" of T' = t1-t0 frames
            if t1 > t0:
                dev = {k: data[k][..., t0:t1].contiguous().to(device) if data[k].dim() == 4
                       else data[k][:, :, :, t0:t1, :].contiguous().to(device) for k in keys}
                mfc = mf[:, :, t0:t1, :].contiguous()
                mbc = mb[:, :, t0:t1, :].contiguous()
                tmp_words = (H * W * (t1 - t0) + 31) // 32
                tmp_f = torch.empty(tmp_words, dtype=torch.int32, device=device)
                tmp_b = torch.empty(tmp_words, dtype=torch.int32, device=device)
                rec_view = records[(t0 - t_begin) * H * W * N.RECORD_FLOATS:]
                N.check(lib.b200_video_pack(N.ptr(dev["frames"]), N.ptr(dev["frames_dx"]), N.ptr(dev["frames_dy"]),
                                            N.ptr(dev["flow_fwd"]), N.ptr(dev["flow_bwd"]), N.ptr(mfc), N.ptr(mbc),
                                            H, W, t1 - t0, 0, t1 - t0, N.ptr(rec_view), N.ptr(tmp_f), N.ptr(tmp_b), st),
                        "b200_video_pack")
                torch.cuda.synchronize(device)
            first = False
            t0 = t1
        # whole-video bitmaps (t_begin == t_end: records untouched)
        dummy = torch.zeros(4, dtype=torch.float32, device=device)
        N.check(lib.b200_video_pack(N.ptr(dummy), N.ptr(dummy), N.ptr(dummy), N.ptr(dummy), N.ptr(dummy),
                                    N.ptr(mf), N.ptr(mb), H, W, T, 0, 0, N.ptr(records), N.ptr(bits_f),
                                    N.ptr(bits_b), st), "b200_video_pack(bitmaps)")
        torch.cuda.synchronize(device)
        return cls(H, W, T, t_begin, t_end, records, bits_f, bits_b)


def video_files(data_folder):
    """The frame files of a video folder in frame order (load_input_data_single's listing)."""
    from pathlib import Path
    data_folder = Path(data_folder)
    return sorted(list(data_folder.glob("*.jpg")) + list(data_folder.glob("*.png")))


def _from_files(cls, data_folder, vid_root, vid_name, resy: int, resx: int, maximum_number_of_frames: int, device,
                filter_optical_flow: bool = True, t_begin: int = 0, t_end: Optional[int] = None,
                decode_all: bool = True):
    """The stage-1 input producer on the device (SURVEY.md §8f rank 1): what `load_input_data_single`
    (unwrap_utils.py:105-163) returns, built frame by frame and pair by pair straight into the pixel records and the
    validity bitmaps — the eight (H, W, ., T) host tensors are never allocated.  The host decodes one image file at
    a time (PIL + the reference's float64 cv2.resize, unwrap_utils.py:124-131) and reads the RAFT .npy flows; the
    differences, the flow resize (cv2.resize-exact, swapped scale factors), the remap-exact forward/backward
    consistency masks and the packing run in libb200deflicker.so (csrc/producer.cu).  Returns (DeviceVideo,
    frames) with `frames` the decoded (H, W, 3, T) fp32 host tensor the PSNR of evaluate.py:740-743 needs.
    With `decode_all` False only the resident frames [t_begin, t_end) are decoded and `frames` is None: a frame
    shard's evaluation reads its frames from the records (DeviceVideo.frame_rgb)."""
    import cv2
    from pathlib import Path
    from PIL import Image
    vid_root = Path(vid_root)
    flow_dir = vid_root / f"{vid_name}_flow"
    files = video_files(data_folder)
    T = int(min(maximum_number_of_frames, len(files)))
    t_end = T if t_end is None else t_end
    lib, st = N.lib(), N.current_stream()
    H, W = int(resy), int(resx)
    HW = H * W
    records = torch.zeros(max(HW * (t_end - t_begin), 1) * N.RECORD_FLOATS, dtype=torch.float32, device=device)
    words = (HW * T + 31) // 32 + 1
    bits_f = torch.zeros(words, dtype=torch.int32, device=device)
    bits_b = torch.zeros(words, dtype=torch.int32, device=device)
    frames = torch.zeros((H, W, 3, T)) if decode_all else None
    pin = torch.zeros(HW * 3, dtype=torch.float32).pin_memory()
    frame_dev = torch.empty(HW * 3, dtype=torch.float32, device=device)
    for i in range(T) if decode_all else range(t_begin, t_end):
        im = np.array(Image.open(str(files[i]))).astype(np.float64) / 255.
        if im.ndim == 2:
            im = np.tile(im[:, :, None], [1, 1, 3])
        fr = torch.from_numpy(cv2.resize(im[:, :, :3], (W, H))).float()        # float64 -> fp32, as the reference's assignment
        if decode_all:
            frames[:, :, :, i] = fr
        if t_begin <= i < t_end:
            pin.copy_(fr.reshape(-1))
            frame_dev.copy_(pin, non_blocking=True)
            N.check(lib.b200_producer_frame(N.ptr(frame_dev), H, W, N.ptr(records[(i - t_begin) * HW * N.RECORD_FLOATS:]),
                                            st), "b200_producer_frame")
            torch.cuda.current_stream().synchronize()                            # `pin` is reused by the next frame
    scratch = torch.empty(int(lib.b200_producer_scratch_floats(H, W)), dtype=torch.float32, device=device)
    for i in range(T - 1):
        a, b = files[i].name, files[i + 1].name
        f12 = np.load(flow_dir / f"{a}_{b}.npy")
        f21 = np.load(flow_dir / f"{b}_{a}.npy")
        if f12.shape[0] < H or f12.shape[1] < W:
            # an up-scaling resize is outside the device kernel's pinned arithmetic: do it as the reference does
            from src.models.stage_1.unwrap_utils import resize_flow
            f12, f21 = resize_flow(f12, newh=H, neww=W), resize_flow(f21, newh=H, neww=W)
        d12 = torch.from_numpy(np.ascontiguousarray(f12, dtype=np.float32)).to(device)
        d21 = torch.from_numpy(np.ascontiguousarray(f21, dtype=np.float32)).to(device)
        resident = (t_begin <= i < t_end) or (t_begin <= i + 1 < t_end)
        N.check(lib.b200_producer_flow_pair(N.ptr(d12), N.ptr(d21), int(f12.shape[0]), int(f12.shape[1]), H, W, T,
                                            t_begin, t_end, N.ptr(records) if resident else None, N.ptr(bits_f),
                                            N.ptr(bits_b), i, 1 if filter_optical_flow else 0, N.ptr(scratch), st),
                "b200_producer_flow_pair")
        torch.cuda.current_stream().synchronize()
    return cls(H, W, T, t_begin, t_end, records, bits_f, bits_b), frames


DeviceVideo.from_files = classmethod(_from_files)


# architecture keys of config_flow_100.json that the fused single-layer step is specialised to
# (src/stage1_neural_atlas.py:112-128 reads them; other values need the generic path: IMLP objects + loss_utils, or
# the segmentation trainer, which takes any IMLP shape)
FUSED_ARCHITECTURE = dict(number_of_layers_mapping1=6, number_of_channels_mapping1=256, use_positional_encoding_mapping1=False,
                          number_of_layers_atlas=8, number_of_channels_atlas=256, positional_encoding_num_atlas=10)
# ... or a mapping on the positional encoding of (x, y, t): use_positional_encoding_mapping1 with
# number_of_positional_encoding_mapping1 frequencies (the tensor-core kernels keep the 6 P columns in one 64-column chunk)
MAPPING_PE_FREQS = range(1, 11)


def mapping_pe_freqs(config: Optional[dict]) -> int:
    """Frequencies of the mapping's positional encoding the config asks for (0: none)."""
    if not config or not config.get("use_positional_encoding_mapping1", False):
        return 0
    return config["number_of_positional_encoding_mapping1"]


def check_architecture(config: dict):
    """Raise instead of silently training a different model than the config describes."""
    bad = {k: config[k] for k, v in FUSED_ARCHITECTURE.items()
           if k in config and config[k] != v and k != "use_positional_encoding_mapping1"}
    if config.get("use_positional_encoding_mapping1", False) is not False:
        pe = config.get("number_of_positional_encoding_mapping1")
        if config["use_positional_encoding_mapping1"] is not True or type(pe) is not int or pe not in MAPPING_PE_FREQS:
            bad["use_positional_encoding_mapping1"] = config["use_positional_encoding_mapping1"]
            bad["number_of_positional_encoding_mapping1"] = pe
    if bad:
        raise N.B200Error(f"the fused stage-1 step is built for {FUSED_ARCHITECTURE} (or use_positional_encoding_mapping1 "
                          f"with number_of_positional_encoding_mapping1 in 1..10); the config asks for {bad}. "
                          "Use the IMLP class + src/models/stage_1/loss_utils.py (any shape) for other architectures.")


class FusedDp:
    """Symmetric (peer-mapped) allocations for b200_dp_adam_step: the parameters, the [gradients || losses] buffer and
    the flag words, with the communicator that names every rank's copies.  torch's symmetric-memory allocator does the
    rendezvous (plumbing); the exchange itself is this library's kernel.  With it a rank keeps the Adam moments of its
    own slice only (gather_moments assembles them)."""

    def __init__(self, pg, device, n_params: int, n_losses: int):
        import torch.distributed as dist
        import torch.distributed._symmetric_memory as symm
        self.pg, self.world = pg, dist.get_world_size(pg)
        self.n_params, self.n_total = n_params, n_params + n_losses
        self.params = symm.empty(n_params, dtype=torch.float32, device=device)
        self.grad_loss = symm.empty(self.n_total, dtype=torch.float32, device=device)
        self.flags = symm.empty(2 * N.MAX_RANKS, dtype=torch.int64, device=device)
        self.params.zero_(); self.grad_loss.zero_(); self.flags.zero_()
        self.handles = [symm.rendezvous(t, pg) for t in (self.grad_loss, self.params, self.flags)]
        self.comm = N.DpComm()
        self.comm.world, self.comm.rank = self.world, dist.get_rank(pg)
        for j in range(self.world):
            self.comm.partials[j] = int(self.handles[0].buffer_ptrs[j])
            self.comm.params[j] = int(self.handles[1].buffer_ptrs[j])
            self.comm.flags[j] = int(self.handles[2].buffer_ptrs[j])
        self.epoch = torch.zeros(1, dtype=torch.int64, device=device)
        torch.cuda.synchronize(device)
        dist.barrier(pg)

    @classmethod
    def create(cls, pg, device, n_params: int, n_losses: int, required: bool) -> Optional["FusedDp"]:
        """The fused optimiser, or None (-> NCCL all-reduce + local Adam) when the allocator is unavailable and
        `required` is false."""
        try:
            return cls(pg, device, n_params, n_losses)
        except Exception as e:                      # noqa: BLE001 - any allocator / rendezvous failure
            if required:
                raise
            import sys
            print(f"b200: fused data-parallel optimiser unavailable ({type(e).__name__}: {e}); "
                  f"using NCCL all-reduce + local Adam", file=sys.stderr)
            return None

    def adam_step(self, exp_avg, exp_avg_sq, lr: float, step_count):
        """reduce-scatter + Adam + all-gather in one kernel (b200_dp_adam_step)."""
        N.check(N.lib().b200_dp_adam_step(C.byref(self.comm), N.ptr(exp_avg), N.ptr(exp_avg_sq), self.n_params,
                                          self.n_total, lr, 0.9, 0.999, 1e-8, N.ptr(step_count), N.ptr(self.epoch),
                                          N.current_stream()), "b200_dp_adam_step")

    def gather_moments(self, exp_avg, exp_avg_sq):
        """Assemble the full Adam moments (checkpoint time) with one all-reduce of the owned slices.  Collective."""
        import torch.distributed as dist
        b, c = C.c_int64(), C.c_int64()
        N.check(N.lib().b200_dp_slice(self.world, self.comm.rank, self.n_total, C.byref(b), C.byref(c)))
        lo, hi = min(b.value, self.n_params), min(b.value + c.value, self.n_params)
        for t in (exp_avg, exp_avg_sq):
            t[:lo].zero_(); t[hi:].zero_()
            dist.all_reduce(t, group=self.pg)


class FlatTrainer:
    """Flat parameters, Adam state, the exchange between ranks and CUDA-graph replay of a stage-1 trainer.

    The networks of NETS share one flat fp32 parameter buffer in that order, which is also the order of the Adam
    parameter groups; `hidden.{i}.weight|bias` are views into it.  Gradients and the loss vector share one buffer
    (`grads`, `losses` are views) so that data parallelism needs ONE exchange: b200_dp_adam_step over symmetric memory
    (FusedDp) with a process group on CUDA when it has more than one rank or `fused_dp` is True (True requires it);
    with `fused_dp` False or a failed set-up, an NCCL all-reduce + the local Adam.

    A subclass calls __init__, sets `cfg`, `descs`, `offsets`, `layouts` (mlp_layout of each network) and `n_params`,
    then calls `_allocate`; it implements `_trip(it)` (one loss_grad of loop trip `it`) and `_regime(it)` (the key of the
    graph that replays that trip)."""

    NETS = ()                   # flat-buffer order = optimiser-group order
    CONSTRUCTION_ORDER = ()     # order the reference script constructs (and so initialises) the networks

    def __init__(self, video: Optional[DeviceVideo], precision: int, device, lr: float, process_group,
                 resx: Optional[int]):
        self.lib = N.lib()
        self.video = video
        self.precision, self.device, self.lr = precision, torch.device(device), lr
        self.resx = resx if resx is not None else (video.W if video is not None else 0)
        self.pg, self.world = process_group, 1
        if process_group is not None:
            import torch.distributed as dist
            self.world = dist.get_world_size(process_group)
        self._ws = None
        self._scratch = {}
        self._graphs = {}

    def _allocate(self, n_losses: int, fused_dp: Optional[bool]):
        dev = self.device
        self._dp = None
        if self.pg is not None and dev.type == "cuda" and fused_dp is not False and (self.world > 1 or fused_dp):
            self._dp = FusedDp.create(self.pg, dev, self.n_params, n_losses, required=bool(fused_dp))
        if self._dp is None:
            self.params = torch.zeros(self.n_params, dtype=torch.float32, device=dev)
            self.grad_loss = torch.zeros(self.n_params + n_losses, dtype=torch.float32, device=dev)
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
        self._pin_loss = torch.zeros(n_losses, dtype=torch.float32).pin_memory() if dev.type == "cuda" else None

    def _scratch_buffer(self, name: str, nbytes: int) -> torch.Tensor:
        """Device scratch kept between calls, replaced by a larger one when a call needs more than `nbytes`."""
        ws = self._scratch.get(name)
        if ws is None or ws.numel() < nbytes:
            ws = self._scratch[name] = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
        return ws

    # ------------------------------------------------------------------ parameters / state dicts
    def _views(self, flat, which):
        w, b, _ = self.layouts[which]
        base = self.offsets[which]
        out = {}
        for i, (k, n) in enumerate(layer_dims(self.descs[which])):
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
        """nn.Linear's default init on the global CPU generator in the script's construction order, weight before
        bias."""
        for which in self.CONSTRUCTION_ORDER:
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
        """Schema of torch.optim.Adam.state_dict() with one group per network of NETS (what evaluate.py stores in the
        checkpoint).  Collective under the fused optimiser: every rank calls it."""
        self.gather_moments()
        state, groups, idx = {}, [], 0
        step = self.step_count.detach().float().cpu().reshape(())
        for which in self.NETS:
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
        for which in self.NETS:
            m, v = self._views(self.exp_avg, which), self._views(self.exp_avg_sq, which)
            for k in m:
                st = sd["state"].get(idx)
                if st is not None:
                    m[k].copy_(st["exp_avg"].to(self.device))
                    v[k].copy_(st["exp_avg_sq"].to(self.device))
                    step = int(st["step"])
                idx += 1
        self.step_count.fill_(step)

    # ------------------------------------------------------------------ optimiser and exchange between ranks
    def adam(self, sl: Optional[slice] = None, m=None, v=None, step=None):
        """b200_adam_step on the slice `sl` of the flat buffers (default: all), with the moments `m`, `v` and the step
        counter `step` instead of the trainer's when given.  The slice's pointers are offsets, not tensor views:
        pre-training calls this every step, and two views would add ~6 us of host time to a host-bound step."""
        sl = slice(0, self.n_params) if sl is None else sl
        at = lambda t: C.c_void_p(t.data_ptr() + 4 * sl.start)        # fp32 element sl.start of a flat buffer
        N.check(self.lib.b200_adam_step(at(self.params), at(self.grads), at(self.exp_avg) if m is None else N.ptr(m),
                                        at(self.exp_avg_sq) if v is None else N.ptr(v), sl.stop - sl.start, self.lr,
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
        self._trip(it)
        if self._dp is not None:
            self.dp_adam()
        else:
            self.all_reduce()
            self.adam()

    def step(self, it: int, use_graph: bool = True):
        """One loop trip on the indices in self.indices (device): losses + gradients, the exchange between ranks (if
        any), then one Adam update of every network (same lr / betas in every group, so one sweep over the flat
        buffer).  On CUDA the trip is captured once per regime in a CUDA graph and replayed.  Returns the device loss
        vector (valid after the stream reaches this point)."""
        if not use_graph or self.device.type != "cuda":
            self._iteration(it)
            return self.losses
        key = self._regime(it)
        g = self._graphs.get(key)
        if g is None:
            # eager warm-up on a side stream (lazy module load, job tables, NCCL channels), state restored afterwards;
            # capture does not execute, so the state is unchanged after it
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

    def step_host(self, inds_cpu: torch.Tensor, it: int, use_graph: bool = True) -> np.ndarray:
        """End-to-end call with HOST buffers: pinned H2D of the index batch, one loop trip,
        D2H of the loss vector (the step's result).  Synchronous."""
        self._pin_inds.copy_(inds_cpu.reshape(-1))
        self.indices.copy_(self._pin_inds, non_blocking=True)
        losses = self.step(it, use_graph)
        self._pin_loss.copy_(losses, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        return self._pin_loss.numpy().copy()

    # ------------------------------------------------------------------ pre-training
    def _pretrain(self, sl: slice, T: int, H: int, W: int, iters: int, generator: Optional[torch.Generator], progress,
                  loss_grad):
        """pre_train_mapping (unwrap_utils.py:176-198) of the network in slice `sl` of the flat buffer: `iters` sweeps
        over the T frames, PRETRAIN_BATCH random pixels of one frame per step, its own Adam(lr=1e-4) with fresh
        moments.  Index draws come from the CPU generator in the reference's order (rows, then columns);
        `loss_grad(f, ys, xs)` makes the native call of frame f on their device copies."""
        n = sl.stop - sl.start
        m = torch.zeros(n, dtype=torch.float32, device=self.device)
        v = torch.zeros_like(m)
        step = torch.zeros(1, dtype=torch.int64, device=self.device)
        ys_d = torch.zeros(PRETRAIN_BATCH, dtype=torch.int64, device=self.device)
        xs_d = torch.zeros_like(ys_d)
        for i in range(iters):
            for f in range(T):
                ys = torch.randint(H, (PRETRAIN_BATCH, 1), generator=generator)
                xs = torch.randint(W, (PRETRAIN_BATCH, 1), generator=generator)
                ys_d.copy_(ys.reshape(-1), non_blocking=True)
                xs_d.copy_(xs.reshape(-1), non_blocking=True)
                loss_grad(f, ys_d, xs_d)
                self.adam(sl, m, v, step)
            if progress:
                progress(i)


class AtlasTrainer(FlatTrainer):
    """Flat parameters/optimiser state of (mapping, atlas) + the fused step."""

    NETS = CONSTRUCTION_ORDER = ("mapping", "atlas")

    def __init__(self, video: Optional[DeviceVideo], config: Optional[dict] = None, precision: int = N.PREC_FP32,
                 device="cuda", lr: float = 1e-4, process_group=None, resx: Optional[int] = None,
                 fused_dp: Optional[bool] = None):
        super().__init__(video, precision, device, lr, process_group, resx)
        self.cfg = dict(DEFAULTS)
        if config:
            self.cfg.update({k: v for k, v in config.items() if k in DEFAULTS})
            check_architecture(config)
        # the mapping of src/stage1_neural_atlas.py:112-119, with the positional encoding the config may ask for
        self.map_desc = make_desc(**dict(MAPPING_DESC, pe_freqs=mapping_pe_freqs(config)))
        self.atlas_desc = make_desc(**ATLAS_DESC)
        self.map_w, self.map_b, self.map_total = mlp_layout(self.map_desc)
        self.atl_w, self.atl_b, self.atl_total = mlp_layout(self.atlas_desc)
        self.n_params = int(self.lib.b200_atlas_param_floats_for(C.byref(self.map_desc)))
        assert self.n_params == self.map_total + self.atl_total
        self.descs = dict(mapping=self.map_desc, atlas=self.atlas_desc)
        self.offsets = dict(mapping=0, atlas=self.map_total)
        self.layouts = dict(mapping=(self.map_w, self.map_b, self.map_total),
                            atlas=(self.atl_w, self.atl_b, self.atl_total))
        self._allocate(N.LOSS_FLOATS, fused_dp)

    def load_state(self, mapping_sd: Dict[str, torch.Tensor], atlas_sd: Dict[str, torch.Tensor]):
        super().load_state(dict(mapping=mapping_sd, atlas=atlas_sd))

    # ------------------------------------------------------------------ native calls
    def _config(self, with_global: bool) -> N.AtlasConfig:
        c = self.cfg
        return N.AtlasConfig(int(c["samples_batch"]), 1 if with_global else 0, self.precision, int(self.resx),
                             float(c["uv_mapping_scale"]), float(c["derivative_amount"]),
                             float(c["global_rigidity_derivative_amount_fg"]), float(c["rgb_coeff"]),
                             float(c["gradient_loss_coeff"]) if c.get("use_gradient_loss", True) else 0.0,
                             float(c["rigidity_coeff"]), float(c["global_rigidity_coeff_fg"]),
                             float(c["optical_flow_coeff"]))

    def _workspace(self):
        if self._ws is None:
            cfg = self._config(True)
            md = C.byref(self.map_desc)
            nbytes = int(self.lib.b200_atlas_workspace_bytes_for(C.byref(cfg), md))
            if cfg.batch < PRETRAIN_BATCH:        # pretrain shares this workspace
                cfg.batch = PRETRAIN_BATCH
                nbytes = max(nbytes, int(self.lib.b200_atlas_workspace_bytes_for(C.byref(cfg), md)))
            if nbytes < 0:
                raise N.B200Error(self.lib.b200_last_error().decode())
            self._ws = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
            self._ws.zero_()
        return self._ws

    def workspace_views(self):
        """Intermediate buffers of the last step as tensor views (tests / debugging): counters, x_map
        [9][cap][4], targets [cap][12], uv [9][cap][2], y_atlas [3][cap][3]."""
        cfg = self._config(True)
        ws = self._workspace()
        off = (C.c_int64 * 8)()
        N.check(self.lib.b200_atlas_workspace_offsets_for(C.byref(cfg), C.byref(self.map_desc), N.ptr(ws), off),
                "b200_atlas_workspace_offsets_for")
        cap = (cfg.batch + 127) // 128 * 128
        f32 = lambda o, n, *shape: ws[o:o + 4 * n].view(torch.float32).view(*shape)
        return dict(cap=cap, counters=ws[off[0]:off[0] + 32].view(torch.int32),
                    x_map=f32(off[2], 9 * cap * 4, 9, cap, 4), targets=f32(off[3], cap * 12, cap, 12),
                    uv=f32(off[6], 9 * cap * 2, 9, cap, 2), y_atlas=f32(off[7], 3 * cap * 3, 3, cap, 3))

    def uses_global(self, it: int) -> bool:
        return bool(self.cfg["include_global_rigidity_loss"]) and it <= self.cfg["stop_global_rigidity"]

    def loss_grad(self, with_global: bool):
        """sampling -> forward -> losses -> backward for the indices currently in self.indices."""
        cfg = self._config(with_global)
        ws = self._workspace()
        N.check(self.lib.b200_atlas_loss_grad_for(C.byref(cfg), C.byref(self.map_desc), C.byref(self.video.struct),
                                                  N.ptr(self.indices), N.ptr(self.params), N.ptr(self.grads),
                                                  N.ptr(self.losses), N.ptr(ws), ws.numel(), N.current_stream()),
                "b200_atlas_loss_grad_for")

    def _trip(self, it: int):
        self.loss_grad(self.uses_global(it))

    def _regime(self, it: int):
        return self.uses_global(it)

    # ------------------------------------------------------------------ pre-training
    def pretrain(self, T: int, H: int, W: int, iters: int, generator: Optional[torch.Generator] = None,
                 progress=None):
        """pre_train_mapping of the mapping block (FlatTrainer._pretrain).  Returns the device loss vector of the last
        step, None when no step ran."""
        larger = max(W, H)
        cfg = self._config(False)
        cfg.batch = PRETRAIN_BATCH
        ws = self._workspace()

        def loss_grad(f, ys, xs):
            N.check(self.lib.b200_pretrain_loss_grad_for(C.byref(cfg), C.byref(self.map_desc), larger, T, f,
                                                         N.ptr(ys), N.ptr(xs), N.ptr(self.params), N.ptr(self.grads),
                                                         N.ptr(self.losses), N.ptr(ws), ws.numel(),
                                                         N.current_stream()), "b200_pretrain_loss_grad_for")
        self._pretrain(self.net_slice("mapping"), T, H, W, iters, generator, progress, loss_grad)
        return self.losses if iters > 0 and T > 0 else None

    # ------------------------------------------------------------------ render / evaluate
    def render_frame(self, f: int, H: int, W: int, T: int, chunk: Optional[int] = None, want_u8: bool = False,
                     precision: Optional[int] = None):
        """Reconstruction of frame f (evaluate.py:644-666): (H, W, 3) fp32 [and uint8 by truncation].  Runs in the
        trainer's precision (tensor cores when the step does); the workspace is kept between calls."""
        prec = self.precision if precision is None else precision
        chunk = H * W if chunk is None else min(chunk, H * W)
        rgb = torch.empty(H * W * 3, dtype=torch.float32, device=self.device)
        u8 = torch.empty(H * W * 3, dtype=torch.uint8, device=self.device) if want_u8 else None
        md = C.byref(self.map_desc)
        ws = self._scratch_buffer("render", int(self.lib.b200_render_workspace_bytes_for(md, chunk)))
        for p0 in range(0, H * W, chunk):
            p1 = min(H * W, p0 + chunk)
            N.check(self.lib.b200_render_for(md, N.ptr(self.params), H, W, T, f, p0, p1, N.ptr(rgb[p0 * 3:]),
                                             N.ptr(u8[p0 * 3:]) if want_u8 else None, prec, N.ptr(ws),
                                             ws.numel(), N.current_stream()), "b200_render_for")
        out = rgb.view(H, W, 3)
        return (out, u8.view(H, W, 3)) if want_u8 else out

    def eval_maps(self, f: int, chunk: Optional[int] = None):
        """Per-pixel maps of frame f that the reference's evaluation dashboards show (evaluate.py:640-700): uv (H, W, 2),
        rigidity loss of every pixel (H, W), forward flow error (H, W; zero where the flow is invalid / last frame)."""
        v = self.video
        H, W = v.H, v.W
        chunk = H * W if chunk is None else min(chunk, H * W)
        uv = torch.empty(H * W * 2, dtype=torch.float32, device=self.device)
        rig = torch.empty(H * W, dtype=torch.float32, device=self.device)
        flow = torch.empty(H * W, dtype=torch.float32, device=self.device)
        ws = self._scratch_buffer("eval", int(self.lib.b200_eval_maps_workspace_bytes(C.byref(self.map_desc), chunk)))
        for p0 in range(0, H * W, chunk):
            p1 = min(H * W, p0 + chunk)
            N.check(self.lib.b200_eval_maps(C.byref(self.map_desc), N.ptr(self.params), C.byref(v.struct), f, p0, p1,
                                            float(self.cfg["derivative_amount"]), float(self.cfg["uv_mapping_scale"]),
                                            self.precision, N.ptr(uv[p0 * 2:]), N.ptr(rig[p0:]), N.ptr(flow[p0:]),
                                            N.ptr(ws), ws.numel(), N.current_stream()), "b200_eval_maps")
        return uv.view(H, W, 2), rig.view(H, W), flow.view(H, W)


def psnr(a: torch.Tensor, b: torch.Tensor) -> float:
    """10 log10(1/MSE) in float64 (skimage peak_signal_noise_ratio, data_range=1; evaluate.py:740-743)."""
    err = torch.mean((a.double() - b.double()) ** 2).item()
    return float(10.0 * math.log10(1.0 / err))


def frame_sse(video: DeviceVideo, f: int, rgb: torch.Tensor, out: Optional[torch.Tensor] = None,
              ws: Optional[torch.Tensor] = None) -> torch.Tensor:
    """b200_frame_sse: float64 sum of (rgb - frame f)^2 over the H*W*3 values, with frame f read from the resident
    records; `rgb` an (H, W, 3) fp32 device tensor.  Returns the 1-element float64 device tensor `out` (valid once the
    stream reaches this point).  `out` and `ws` (b200_frame_sse_workspace_bytes) may be passed for graph capture."""
    lib = N.lib()
    rgb = rgb.contiguous()
    if rgb.dtype != torch.float32 or rgb.numel() != video.H * video.W * 3 or rgb.device.type != "cuda":
        raise N.B200Error(f"rgb must be an fp32 ({video.H}, {video.W}, 3) device tensor")
    if out is None:
        out = torch.empty(1, dtype=torch.float64, device=rgb.device)
    if ws is None:
        ws = torch.empty(int(lib.b200_frame_sse_workspace_bytes(video.H, video.W)), dtype=torch.uint8, device=rgb.device)
    N.check(lib.b200_frame_sse(C.byref(video.struct), int(f), N.ptr(rgb), N.ptr(out), N.ptr(ws), ws.numel(),
                               N.current_stream()), "b200_frame_sse")
    return out


def psnr_device(video: DeviceVideo, f: int, rgb: torch.Tensor) -> float:
    """psnr(frame f, rgb) with the squared error summed on the device against frame f's resident records."""
    sse = float(frame_sse(video, f, rgb).item())
    return float(10.0 * math.log10(1.0 / (sse / (video.H * video.W * 3))))


def frame_range(rank: int, world: int, T: int):
    """Contiguous frame block owned by `rank` (SURVEY §8e): [t_begin, t_end)."""
    base, rem = divmod(T, world)
    t0 = rank * base + min(rank, rem)
    return t0, t0 + base + (1 if rank < rem else 0)
