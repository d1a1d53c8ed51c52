"""Fidelity of frame sequences to a reference on the device (b200_fidelity; DESIGN §4f): SSIM and PSNR of each frame
against the reference frame at the same position.

For a frame O and its reference R (resized to O's size when they differ), the kernel sums SSIM over O's interior
pixels (5 <= x < W - 5, 5 <= y < H - 5) and channels, and the squared error over all of O's values; S(t) and PSNR(t)
follow from the sums (`frame_values`).  `FidelityScorer` scores every requested sequence on a window of frames, one
call per 32 frame pairs."""
from __future__ import annotations

import math
import time
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _native as N
from .flicker import PIXEL_BITS

RADIUS = 5


def frame_desc(frame: torch.Tensor, ref: torch.Tensor) -> N.FidelityFrame:
    """The descriptor of one frame and its reference: (H, W, 3) and (Hr, Wr, 3) uint8 / uint16 contiguous device
    tensors (each its own type) that stay alive until the call's work has run."""
    for name, t in (("frame", frame), ("ref", ref)):
        if t.device.type != "cuda" or not t.is_contiguous():
            raise N.B200Error(f"{name} must be a contiguous device tensor")
        if t.dtype not in PIXEL_BITS:
            raise N.B200Error(f"{name} must be uint8 or uint16 (got {t.dtype})")
        if t.dim() != 3 or t.shape[2] != 3:
            raise N.B200Error(f"{name} must be an (H, W, 3) image (got {tuple(t.shape)})")
    return N.FidelityFrame(frame.data_ptr(), ref.data_ptr(), frame.shape[0], frame.shape[1], ref.shape[0],
                           ref.shape[1], PIXEL_BITS[frame.dtype], PIXEL_BITS[ref.dtype])


def workspace_bytes(descs: Sequence[N.FidelityFrame]) -> int:
    table = (N.FidelityFrame * len(descs))(*descs)
    nb = int(N.lib().b200_fidelity_workspace_bytes(table, len(descs)))
    if nb < 0:
        raise N.B200Error("b200_fidelity_workspace_bytes: " + N.last_error())
    return nb


def fidelity(descs: Sequence[N.FidelityFrame], sums: torch.Tensor, ws: torch.Tensor,
             ssim_map: Optional[torch.Tensor] = None):
    """One b200_fidelity call on the current stream: sums [n][2] float64 (SSIM sum over the interior, squared-error
    sum) and, when given, the per-pixel, per-channel SSIM (fp32, NaN outside the interior), frame after frame."""
    table = (N.FidelityFrame * len(descs))(*descs)
    N.check(N.lib().b200_fidelity(table, len(descs), N.ptr(sums), N.ptr(ssim_map), N.ptr(ws), ws.numel(),
                                  N.current_stream()), "b200_fidelity")


def frame_values(ssim_sum: float, sse: float, H: int, W: int) -> Tuple[float, Optional[float]]:
    """S(t) and PSNR(t) of an H x W frame from its sums; PSNR is None for a frame equal to its reference."""
    s = float(ssim_sum) / (3.0 * (H - 2 * RADIUS) * (W - 2 * RADIUS))
    if sse == 0:
        return s, None
    return s, 10.0 * math.log10(1.0 / (float(sse) / (3.0 * H * W)))


class FidelityScorer:
    """Owns the device workspace, the sums and the pinned staging of one process's scoring."""

    def __init__(self, device):
        self.device = torch.device(device)
        self.ws = torch.empty(0, dtype=torch.uint8, device=self.device)
        self.sums = torch.empty(N.FIDELITY_MAX_FRAMES, 2, dtype=torch.float64, device=self.device)
        self.pinned: Dict[str, torch.Tensor] = {}
        self.device_seconds = 0.0

    def _upload(self, name: str, arrays: List[np.ndarray]) -> torch.Tensor:
        """The arrays (one shape and dtype) as one device tensor, through the pinned buffer `name`."""
        shape, dt = (len(arrays),) + arrays[0].shape, torch.from_numpy(arrays[0][:0]).dtype
        n = int(np.prod(shape)) * arrays[0].itemsize
        buf = self.pinned.get(name)
        if buf is None or buf.numel() < n:
            buf = self.pinned[name] = torch.empty(n, dtype=torch.uint8, pin_memory=True)
        host = buf[:n].view(dt).view(shape)
        hn = host.numpy()
        for i, a in enumerate(arrays):
            hn[i] = a
        return host.to(self.device, non_blocking=True)

    def score_frames(self, refs: List[np.ndarray],
                     frames: Dict[str, List[np.ndarray]]) -> Dict[str, List[Tuple[float, float]]]:
        """refs: the window's reference frames; frames: per sequence its frames of the window (frame i is scored
        against refs[i]; a sequence may have fewer).  Returns per sequence the (SSIM sum, squared-error sum) of its
        frames in order."""
        t0 = time.perf_counter()
        out: Dict[str, List[Tuple[float, float]]] = {name: [] for name in frames}
        if not refs:
            return out
        ref = self._upload("ref", refs)
        # the descriptors hold raw pointers: every upload stays referenced until the calls below have run
        resident = [ref]
        jobs, descs = [], []
        for si, (name, fr) in enumerate(frames.items()):
            k = min(len(fr), len(refs))
            if k == 0:
                continue
            dev = self._upload("frames%d" % si, fr[:k])
            resident.append(dev)
            for i in range(k):
                jobs.append(name)
                descs.append(frame_desc(dev[i], ref[i]))
        for c0 in range(0, len(descs), N.FIDELITY_MAX_FRAMES):
            chunk = descs[c0:c0 + N.FIDELITY_MAX_FRAMES]
            nb = workspace_bytes(chunk)
            if self.ws.numel() < nb:
                self.ws = torch.empty(nb, dtype=torch.uint8, device=self.device)
            fidelity(chunk, self.sums, self.ws)
            host = self.sums[:len(chunk)].cpu().numpy()             # synchronises: the staging may be reused
            for name, (s, e) in zip(jobs[c0:c0 + N.FIDELITY_MAX_FRAMES], host):
                out[name].append((float(s), float(e)))
        torch.cuda.synchronize(self.device)
        del resident
        self.device_seconds += time.perf_counter() - t0
        return out
