#!/usr/bin/env python
"""A few stage-2 frames (UNet + TransformNet at 1088x1920, wgmma convolutions) — for launch lists."""
import os
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "all-in-one-deflicker_b200"))
from b200 import nn as K  # noqa: E402
from src.models.network_filter import UNet  # noqa: E402
from src.models.network_local import TransformNet  # noqa: E402

K.set_conv_precision("tc")
g = torch.Generator().manual_seed(0)
unet = UNet(6, 3, 32).cuda().eval()
tn = TransformNet(types.SimpleNamespace(nf=32, norm="IN", model="TransformNet", blocks=5), 12, 3).cuda().eval()
x6 = torch.rand(1, 6, 1088, 1920, generator=g).cuda()
x12 = torch.rand(1, 12, 1088, 1920, generator=g).cuda()
with torch.no_grad():
    for _ in range(int(sys.argv[1]) if len(sys.argv) > 1 else 3):
        unet(x6); tn(x12, None)
torch.cuda.synchronize()
