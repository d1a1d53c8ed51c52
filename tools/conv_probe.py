#!/usr/bin/env python
"""A few single convolutions at stage-2 sizes on the wgmma path (for ncu captures)."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "all-in-one-deflicker_b200"))
from b200 import nn as K  # noqa: E402

K.set_conv_precision("tc")
g = torch.Generator().manual_seed(0)
cases = [(6, 32, 3, 1088, 1920, "zeros", 1), (32, 32, 3, 1088, 1920, "zeros", 1), (128, 128, 3, 272, 480, "zeros", 1),
         (128, 128, 3, 272, 480, "reflect", 1), (128, 32, 3, 544, 960, "reflect", 2), (64, 3, 7, 1088, 1920, "reflect", 1)]
sel = [int(v) for v in sys.argv[1:]] or range(len(cases))
for cin, cout, k, h, w, mode, up in [cases[i] for i in sel]:
    x = torch.randn(1, cin, h, w, generator=g).cuda()
    wt = (torch.randn(cout, cin, k, k, generator=g) / (cin * k * k) ** 0.5).cuda()
    b = torch.zeros(cout).cuda()
    for _ in range(2):
        K.conv2d(x, wt, b, pad=k // 2, pad_mode=mode, act="relu", upsample=up)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    K.conv2d(x, wt, b, pad=k // 2, pad_mode=mode, act="relu", upsample=up)
    e1.record()
    torch.cuda.synchronize()
    print(cin, cout, k, h, w, mode, up, "ms", round(e0.elapsed_time(e1), 4))
