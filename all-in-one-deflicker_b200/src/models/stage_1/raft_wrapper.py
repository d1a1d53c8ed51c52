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

    def load_image(self, fn):
        """uint8 image file -> (3, H, W) float tensor in [0, 255], downsampled when its long edge is too large."""
        pixels = np.array(Image.open(fn), dtype=np.uint8)
        rows, cols = pixels.shape[:2]
        shrink = max(rows, cols) / self.args.max_long_edge
        if shrink > 1:
            pixels = cv2.resize(pixels, (int(cols // shrink), int(rows // shrink)), interpolation=cv2.INTER_AREA)
        return torch.from_numpy(pixels).permute(2, 0, 1).float()

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
