#!/usr/bin/env python
"""Per-convolution CUDA-event times of the update block, UNet and TransformNet at the aux-bench sizes, for
both convolution arithmetics.  Diagnostic only (synchronises around every call)."""
import inspect
import json
import os
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "all-in-one-deflicker_b200"))


def main():
    from b200 import nn as K
    from src.models.network_filter import UNet
    from src.models.network_local import TransformNet
    from src.models.stage_1.core.update import BasicUpdateBlock
    dev = "cuda"
    rows = []
    orig = K.conv2d

    sig = inspect.signature(orig)

    def timed_conv(x, w, *a, **kw):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        y = orig(x, w, *a, **kw)
        e1.record()
        torch.cuda.synchronize()
        # the output geometry comes from the arguments: a chained producer with keep_fp32=False returns None
        p = sig.bind(x, w, *a, **kw)
        p.apply_defaults()
        p = p.arguments
        chained_in = isinstance(x, K.Chain)
        n, h, wd = (x.n, x.h, x.w) if chained_in else (x.shape[0], x.shape[2], x.shape[3])
        ph, pw = (p["pad"], p["pad"]) if isinstance(p["pad"], int) else p["pad"]
        cout, cin, kh, kw = w.shape
        oh = (h * p["upsample"] + 2 * ph - kh) // p["stride"] + 1
        ow = (wd * p["upsample"] + 2 * pw - kw) // p["stride"] + 1
        macs = n * oh * ow * cout * cin * kh * kw
        ms = e0.elapsed_time(e1)
        rows.append({"net": tag[0], "prec": K.conv_precision(), "cin": cin, "cout": cout, "k": [kh, kw],
                     "out_hw": [oh, ow], "pad": p["pad_mode"], "up": p["upsample"], "stride": p["stride"],
                     "chained_in": chained_in, "chain_out": p["chain_out"] is not None, "ms": round(ms, 4),
                     "tflops": round(2 * macs / ms / 1e9, 1)})
        return y

    K.conv2d = timed_conv
    tag = [""]
    g = torch.Generator().manual_seed(0)
    h8, w8 = 135, 240
    ub = BasicUpdateBlock(types.SimpleNamespace(corr_levels=4, corr_radius=4), hidden_dim=128).to(dev)
    net = torch.tanh(torch.randn(1, 128, h8, w8, generator=g)).to(dev)
    inp = torch.relu(torch.randn(1, 128, h8, w8, generator=g)).to(dev)
    flow = torch.randn(1, 2, h8, w8, generator=g).to(dev)
    corr = torch.randn(1, 324, h8, w8, generator=g).to(dev)
    unet = UNet(6, 3, 32).to(dev).eval()
    tn = TransformNet(types.SimpleNamespace(nf=32, norm="IN", model="TransformNet", blocks=5), 12, 3).to(dev).eval()
    x6 = torch.rand(1, 6, 1088, 1920, generator=g).to(dev)
    x12 = torch.rand(1, 12, 1088, 1920, generator=g).to(dev)
    for prec in sys.argv[1:] or ["tc"]:
        K.set_conv_precision(prec)
        for rep in range(2):
            rows.clear()
            tag[0] = "update"; ub(net, inp, corr, flow)
            tag[0] = "unet"; unet(x6)
            tag[0] = "tn"; tn(x12, None)
        for r in rows:
            print(json.dumps(r))
        for name in ("update", "unet", "tn"):
            print(name, prec, "conv total ms", round(sum(r["ms"] for r in rows if r["net"] == name), 3))


if __name__ == "__main__":
    main()
