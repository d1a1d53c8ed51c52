"""Temporal warping error of frame sequences on the device (b200_warp_error; DESIGN §4e).

For consecutive frames t, t+1 and the flow pre-pass's flows F = `<t>_<t+1>.npy`, B = `<t+1>_<t>.npy`, the kernel sums
sum_c (O_t(p, c) - O_{t+1}(p + F(p), c))^2 over the pixels p whose match lies in the frame and passes the
forward-backward occlusion test, and counts them; E(t) = sum / (3 |M|).  `FlickerScorer` scores every requested
sequence on a pair while that pair's flows are resident, a window of consecutive pairs per call."""
from __future__ import annotations

import time
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _native as N

PIXEL_BITS = {torch.uint8: 8, torch.uint16: 16}


def pair_desc(f0: torch.Tensor, f1: torch.Tensor, fwd: torch.Tensor, bwd: torch.Tensor) -> N.WarpPair:
    """The descriptor of one pair: frames (H, W, 3) uint8 / uint16 and flows (Hf, Wf, 2) fp32, contiguous device
    tensors that stay alive until the call's work has run."""
    for name, t in (("frame0", f0), ("frame1", f1), ("fwd", fwd), ("bwd", bwd)):
        if t.device.type != "cuda" or not t.is_contiguous():
            raise N.B200Error(f"{name} must be a contiguous device tensor")
    if f0.dtype not in PIXEL_BITS or f1.dtype != f0.dtype:
        raise N.B200Error(f"frames must both be uint8 or both uint16 (got {f0.dtype} and {f1.dtype})")
    if f0.dim() != 3 or f0.shape[2] != 3 or f1.shape != f0.shape:
        raise N.B200Error(f"frames must be two (H, W, 3) images of one size (got {tuple(f0.shape)}, {tuple(f1.shape)})")
    if fwd.dtype != torch.float32 or fwd.dim() != 3 or fwd.shape[2] != 2 or bwd.shape != fwd.shape or bwd.dtype != fwd.dtype:
        raise N.B200Error(f"flows must be two (Hf, Wf, 2) fp32 arrays of one size (got {tuple(fwd.shape)}, "
                          f"{tuple(bwd.shape)})")
    return N.WarpPair(f0.data_ptr(), f1.data_ptr(), fwd.data_ptr(), bwd.data_ptr(), f0.shape[0], f0.shape[1],
                      fwd.shape[0], fwd.shape[1], PIXEL_BITS[f0.dtype], 0)


def workspace_bytes(descs: Sequence[N.WarpPair]) -> int:
    table = (N.WarpPair * len(descs))(*descs)
    nb = int(N.lib().b200_warp_error_workspace_bytes(table, len(descs)))
    if nb < 0:
        raise N.B200Error("b200_warp_error_workspace_bytes: " + N.last_error())
    return nb


def warp_error(descs: Sequence[N.WarpPair], sums: torch.Tensor, ws: torch.Tensor, error: Optional[torch.Tensor] = None,
               mask: Optional[torch.Tensor] = None):
    """One b200_warp_error call on the current stream: sums [n][2] float64 (masked squared-error sum, |M|), and, when
    given, the per-pixel error (fp32) and mask (uint8), pair after pair."""
    table = (N.WarpPair * len(descs))(*descs)
    N.check(N.lib().b200_warp_error(table, len(descs), N.ptr(sums), N.ptr(error), N.ptr(mask), N.ptr(ws), ws.numel(),
                                    N.current_stream()), "b200_warp_error")


def pair_value(sse: float, count: float) -> float:
    """E(t) of a pair from its sums: NaN for an empty mask."""
    return float(sse) / (3.0 * float(count)) if count > 0 else float("nan")


class FlickerScorer:
    """Owns the device workspace and the pinned staging of one process's scoring.  `score_window` takes a window of
    consecutive pairs: each pair's two flows once, and for each sequence the window's frames once."""

    def __init__(self, device):
        self.device = torch.device(device)
        self.ws = torch.empty(0, dtype=torch.uint8, device=self.device)
        self.sums = torch.empty(N.WARP_MAX_PAIRS, 2, dtype=torch.float64, device=self.device)
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

    def score_window(self, flows: List[Tuple[np.ndarray, np.ndarray]],
                     frames: Dict[str, List[np.ndarray]]) -> Dict[str, List[Tuple[float, float]]]:
        """flows: (F, B) of the window's k pairs; frames: per sequence its frames of the window, k + 1 of them, or
        fewer when the sequence ends inside the window (a pair is scored when both of its frames are there).  Returns
        per sequence the (squared-error sum, |M|) of its pairs in order."""
        t0 = time.perf_counter()
        fwd = self._upload("fwd", [f for f, _ in flows])
        bwd = self._upload("bwd", [b for _, b in flows])
        # the descriptors hold raw pointers: every upload must stay referenced until the calls below have run, or the
        # caching allocator hands its memory to the next upload
        resident = [fwd, bwd]
        jobs, descs = [], []
        for si, (name, fr) in enumerate(frames.items()):
            if len(fr) < 2:
                continue
            dev = self._upload("frames%d" % si, fr)
            resident.append(dev)
            for i in range(min(len(flows), len(fr) - 1)):
                jobs.append(name)
                descs.append(pair_desc(dev[i], dev[i + 1], fwd[i], bwd[i]))
        out: Dict[str, List[Tuple[float, float]]] = {name: [] for name in frames}
        for c0 in range(0, len(descs), N.WARP_MAX_PAIRS):
            chunk = descs[c0:c0 + N.WARP_MAX_PAIRS]
            nb = workspace_bytes(chunk)
            if self.ws.numel() < nb:
                self.ws = torch.empty(nb, dtype=torch.uint8, device=self.device)
            warp_error(chunk, self.sums, self.ws)
            host = self.sums[:len(chunk)].cpu().numpy()             # synchronises: the staging may be reused
            for name, (sse, cnt) in zip(jobs[c0:c0 + N.WARP_MAX_PAIRS], host):
                out[name].append((float(sse), float(cnt)))
        torch.cuda.synchronize(self.device)
        del resident
        self.device_seconds += time.perf_counter() - t0
        return out
