"""Stage 2 (neural filter + local refinement) from frames to frames, with the frames kept on the device.

`Stage2.frame(content, atlas)` is one trip of the loop of src/neural_filter_and_refinement.py: 8-bit images in, the
three 8-bit images the script writes out.  The filter network's input is built by b200_stage2_pack_input and the output
images by b200_stage2_emit (csrc/stage2_io.cu); only uint8 crosses the bus, through pinned buffers.  The arithmetic is
the script's, restated from OpenCV's own resize code (oracle/stage2_io_oracle.py); images that are not 8-bit go through
the host arithmetic of src/models/utils.py instead.
"""
from __future__ import annotations

import numpy as np
import torch

from . import _native as N


def pad_geometry(h: int, w: int):
    """(left, right, top, bottom) replicate padding of an (h, w) frame, as src/models/utils.py InputPadder has it."""
    ph, pw = -h % 32, -w % 32
    return pw // 2, pw - pw // 2, 0, ph


def pack_input(content, atlas, out=None):
    """[1, 6, Hp, Wp] fp32 filter-network input from two contiguous uint8 device images (H, W) or (H, W, 1 | 3 | 4)."""
    for t in (content, atlas):
        if not (t.is_cuda and t.dtype == torch.uint8 and t.is_contiguous() and t.dim() in (2, 3)):
            raise N.B200Error("pack_input takes contiguous uint8 CUDA images (H, W[, C])")
    hc, wc = content.shape[:2]
    if out is None:
        left, right, _, bottom = pad_geometry(hc, wc)
        out = torch.empty(1, 6, hc + bottom, wc + left + right, device=content.device)
    if not (out.is_cuda and out.dtype == torch.float32 and out.is_contiguous() and out.dim() == 4 and out.shape[:2] == (1, 6)):
        raise N.B200Error("pack_input writes a contiguous [1, 6, Hp, Wp] fp32 CUDA tensor")
    hp, wp = out.shape[2:]                         # checked against the content's size by the library
    chans = lambda t: 1 if t.dim() == 2 else t.shape[2]
    N.check(N.lib().b200_stage2_pack_input(N.ptr(content), hc, wc, chans(content), N.ptr(atlas), atlas.shape[0],
                                           atlas.shape[1], chans(atlas), N.ptr(out), hp, wp, N.current_stream()),
            "b200_stage2_pack_input")
    return out


def emit(t, out, x_off: int, w: int):
    """Writes channels of t ([1, 3, Hp, Wp] fp32 CUDA, a channel slice of a contiguous tensor is fine) as the uint8 BGR
    image save_img would write after cv2.resize(tensor2img(t), (w, out rows)), into columns [x_off, x_off + w) of the
    uint8 CUDA image `out` (H, Wtotal, 3)."""
    if not (t.is_cuda and t.dtype == torch.float32 and t.dim() == 4 and t.shape[:2] == (1, 3)
            and t.stride(3) == 1 and t.stride(2) == t.shape[3]):
        raise N.B200Error("emit takes a [1, 3, Hp, Wp] fp32 CUDA tensor with dense planes")
    if not (out.is_cuda and out.dtype == torch.uint8 and out.is_contiguous() and out.dim() == 3 and out.shape[2] == 3
            and 0 <= x_off and x_off + w <= out.shape[1]):
        raise N.B200Error("emit writes into a contiguous uint8 CUDA image (H, W, 3)")
    N.check(N.lib().b200_stage2_emit(N.ptr(t), t.stride(1), t.shape[2], t.shape[3], N.ptr(out), 3 * x_off,
                                     3 * out.shape[1], out.shape[0], w, N.current_stream()), "b200_stage2_emit")


def host_input(content, atlas, device):
    """The filter network's input by the host arithmetic of src/models/utils.py (load_image after the decode,
    InputPadder.pad, cat) — for decoded images that are not 8-bit."""
    import cv2
    from src.models.utils import InputPadder

    def unit(a):
        a = np.asarray(a) / 255.
        return np.repeat(a[:, :, None], 3, axis=2) if a.ndim == 2 else a[..., :3]
    c, a = unit(content), unit(atlas)
    a = cv2.resize(a, (c.shape[1], c.shape[0]), cv2.INTER_LINEAR)
    c, a = (torch.from_numpy(v).permute(2, 0, 1).unsqueeze(0).to(device, dtype=torch.float) for v in (c, a))
    return torch.cat(InputPadder(c.shape).pad(c, a), dim=1)


class Stage2:
    """The two networks and every device / pinned buffer of one frame geometry (re-made when the geometry changes).

    frame() returns {"filter", "final": uint8 BGR (H, W, 3), "concat": (H, 3 W, 3)} as numpy views of one of two
    pinned buffers used in turn: a result stays valid until the call after next."""

    def __init__(self, filter_net, local_net, device):
        self.filter_net, self.local_net, self.device = filter_net, local_net, torch.device(device)
        self._geom = None
        self.reset()

    def reset(self):
        """Forget the previous frame: the next frame() is a first frame."""
        self._o1 = self._p1 = None

    def _buffers(self, geom):
        if geom == self._geom:
            return
        (hc, wc, cc), (hs, ws, cs) = geom
        dev = self.device
        self._stage = [torch.empty(s, dtype=torch.uint8).pin_memory() for s in ((hc, wc, cc), (hs, ws, cs))]
        self._u8 = [torch.empty(s, dtype=torch.uint8, device=dev) for s in ((hc, wc, cc), (hs, ws, cs))]
        left, right, _, bottom = pad_geometry(hc, wc)
        self._x6 = torch.empty(1, 6, hc + bottom, wc + left + right, device=dev)
        # the three images of one frame, back to back: concat (H, 3W, 3), filter (H, W, 3), final (H, W, 3)
        n = hc * wc * 3
        self._out = torch.empty(5 * n, dtype=torch.uint8, device=dev)
        self._host = [torch.empty(5 * n, dtype=torch.uint8).pin_memory() for _ in range(2)]
        self._done = [torch.cuda.Event() for _ in range(2)]
        self._turn = 0
        self._geom = geom

    def _to_device(self, img, k):
        if torch.is_tensor(img) and img.is_cuda:
            return img.contiguous()
        src = img if torch.is_tensor(img) else torch.from_numpy(np.ascontiguousarray(img))
        self._stage[k].copy_(src.reshape(self._stage[k].shape))
        self._u8[k].copy_(self._stage[k], non_blocking=True)
        return self._u8[k]

    @torch.no_grad()
    def frame(self, content, atlas):
        is_u8 = lambda a: (a.dtype == torch.uint8) if torch.is_tensor(a) else (np.asarray(a).dtype == np.uint8)
        shape3 = lambda a: tuple(a.shape) + (1,) * (3 - len(a.shape))
        hc, wc = content.shape[:2]
        with torch.cuda.device(self.device):
            self._buffers((shape3(content), shape3(atlas)))
            if is_u8(content) and is_u8(atlas):
                x6 = pack_input(self._to_device(content, 0), self._to_device(atlas, 1), out=self._x6)
            else:
                as_np = lambda a: a.cpu().numpy() if torch.is_tensor(a) else a
                x6 = host_input(as_np(content), as_np(atlas), self.device)
            pred = self.filter_net(x6)
            if self._o1 is None:
                o2 = pred
            else:
                out, _ = self.local_net(torch.cat((pred, self._o1, pred, self._p1), dim=1), None)
                o2 = pred + out
            self._p1, self._o1 = pred, o2
            n = hc * wc * 3
            concat, filt, final = (self._out[a:b].view(hc, -1, 3) for a, b in ((0, 3 * n), (3 * n, 4 * n), (4 * n, 5 * n)))
            for k, t in enumerate((x6[:, 0:3], x6[:, 3:6], pred)):
                emit(t, concat, k * wc, wc)
            emit(pred, filt, 0, wc)
            emit(o2, final, 0, wc)
            host, done = self._host[self._turn], self._done[self._turn]
            self._turn ^= 1
            host.copy_(self._out, non_blocking=True)
            done.record()
            done.synchronize()
        h = host.numpy()
        return {"concat": h[:3 * n].reshape(hc, 3 * wc, 3), "filter": h[3 * n:4 * n].reshape(hc, wc, 3),
                "final": h[4 * n:].reshape(hc, wc, 3)}
