"""`RAFTWrapper` — the object `preprocess_optical_flow.py` drives, with the reference's constructor and method
names (src/models/stage_1/raft_wrapper.py:16-73).  Checkpoints saved from `nn.DataParallel` (keys prefixed with
`module.`) load directly; frames whose long edge exceeds `max_long_edge` are area-downsampled first; inputs are
padded to multiples of 8 and refined for 20 iterations, as in the reference."""
import argparse

import cv2
import numpy as np
import torch
from PIL import Image

from src.models.stage_1.core.raft import RAFT
from src.models.stage_1.core.utils.utils import InputPadder

device = torch.device("cuda")      # the current device: cuda:LOCAL_RANK on a rank of a multi-GPU pre-pass
REFINEMENT_ITERS = 20


def _strip_data_parallel(state_dict):
    return {(k[7:] if k.startswith("module.") else k): v for k, v in state_dict.items()}


def _to_hw2(flow):
    return flow[0].permute(1, 2, 0).detach().cpu().numpy()


class RAFTWrapper():
    def __init__(self, model_path, max_long_edge=900):
        self.args = argparse.Namespace(small=False, mixed_precision=True, model=model_path, max_long_edge=max_long_edge)
        self.model = RAFT(self.args)
        if model_path is not None:
            self.model.load_state_dict(_strip_data_parallel(torch.load(model_path, map_location="cpu")))
        self.model.to(device).eval()

    def _decoded_size(self, rows, cols):
        """(rows, cols) of a frame of rows x cols pixels after the long-edge downsampling of load_image."""
        shrink = max(rows, cols) / self.args.max_long_edge
        return (int(rows // shrink), int(cols // shrink)) if shrink > 1 else (rows, cols)

    def load_image(self, fn):
        """uint8 image file -> (3, H, W) float tensor in [0, 255], downsampled when its long edge is too large."""
        pixels = np.array(Image.open(fn), dtype=np.uint8)
        rows, cols = pixels.shape[:2]
        size = self._decoded_size(rows, cols)
        if size != (rows, cols):
            pixels = cv2.resize(pixels, (size[1], size[0]), interpolation=cv2.INTER_AREA)
        return torch.from_numpy(pixels).permute(2, 0, 1).float()

    def feature_grid(self, fn):
        """(H8, W8): RAFT's feature-map size for frames like image file `fn` (read from its header)."""
        with Image.open(fn) as im:
            cols, rows = im.size
        rows, cols = self._decoded_size(rows, cols)
        return (rows + 7) // 8, (cols + 7) // 8

    def load_window(self, image_files):
        """Consecutive frames, in the given order -> one (N, 3, H, W) float host tensor; compute_flow_sequence moves it
        to the device and pads it.  Runs on a decoder thread, so it makes no CUDA call: one from another thread would
        invalidate a CUDA graph being captured."""
        return torch.stack([self.load_image(f) for f in image_files], dim=0)

    def load_image_list(self, image_files):
        """Sorted file names -> one (N, 3, H, W) batch on the device, padded to multiples of 8."""
        batch = torch.stack([self.load_image(f) for f in sorted(image_files)], dim=0).to(device)
        batch, = InputPadder(batch.shape).pad(batch)
        return batch

    def load_images(self, fn1, fn2):
        pair = self.load_image_list([fn1, fn2])
        return pair[0:1], pair[1:2]

    def _padded(self, im1, im2):
        return InputPadder(im1.shape).pad(im1, im2)

    def compute_flow(self, im1, im2):
        a, b = self._padded(im1, im2)
        _, up = self.model(a, b, iters=REFINEMENT_ITERS, test_mode=True)
        return _to_hw2(up)

    def compute_flow_both(self, im1, im2):
        """(flow 1->2, flow 2->1): what two compute_flow calls return, with the feature encoder run once."""
        a, b = self._padded(im1, im2)
        (_, up12), (_, up21) = self.model.forward_both(a, b, iters=REFINEMENT_ITERS)
        return _to_hw2(up12), _to_hw2(up21)

    def compute_flow_sequence(self, frames, pad_to=None):
        """N consecutive frames from load_window -> (forward flows, backward flows), each an (N - 1, H, W, 2) float32
        array: [k] is what compute_flow_both returns for frames k and k + 1, bit for bit.  `pad_to`: see
        RAFT.forward_sequence.  The flows come back through pinned host memory."""
        batch = frames.to(device)
        batch, = InputPadder(batch.shape).pad(batch)
        (_, up_fwd), (_, up_bwd) = self.model.forward_sequence(batch, iters=REFINEMENT_ITERS, pad_to=pad_to)
        flows = torch.cat([up_fwd, up_bwd]).permute(0, 2, 3, 1).contiguous()
        host = torch.empty(flows.shape, dtype=flows.dtype, pin_memory=True)
        host.copy_(flows, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        k = up_fwd.shape[0]
        out = host.numpy()
        return out[:k], out[k:]
