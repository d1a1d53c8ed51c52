#!/usr/bin/env python
"""CUDA-event times of TransformNet's ConvLSTM gate layer alone at the 1088x1920 stage-2 geometry (gates at 272 x 480,
C = 128, N = 1), on the wgmma path: the fused layer (b200_convlstm_tma, cell update in the epilogue) against the
gate convolution writing the 512-channel gates tensor followed by the cell kernel, with and without a previous state,
for a chained (pre-packed) input as TransformNet runs it and a plain fp32 input.  Median of --reps timed calls after
--warmup; prints one JSON line per variant.

    python tools/convlstm_rate.py [--reps 50] [--warmup 10] [--dump-stateless PATH]

--dump-stateless PATH writes TransformNet(X, None)'s output on a seeded 1088x1920 input (wgmma path) to PATH, so two
builds can be compared bit for bit."""
import argparse
import ctypes as C
import json
import os
import statistics
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "all-in-one-deflicker_b200"))


def _time(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    ms = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    return statistics.median(ms), min(ms)


def dump_stateless(path):
    from b200 import nn as K
    from src.models.network_local import TransformNet
    torch.manual_seed(0)
    tn = TransformNet(types.SimpleNamespace(nf=32, norm="IN", model="TransformNet", blocks=5), 12, 3).cuda().eval()
    g = torch.Generator().manual_seed(1)
    x = torch.rand(1, 12, 1088, 1920, generator=g).cuda()
    K.set_conv_precision("tc")
    y, (h, c) = tn(x, None)
    torch.save({"y": y.cpu(), "hidden": h.cpu(), "cell": c.cpu()}, path)
    print(json.dumps({"dumped": path}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--dump-stateless", default=None)
    args = ap.parse_args()
    if args.dump_stateless:
        dump_stateless(args.dump_stateless)
        return
    from b200 import _native as N
    from b200 import nn as K
    dev = "cuda"
    n, c, h, w = 1, 128, 272, 480
    g = torch.Generator().manual_seed(0)
    x = torch.randn(n, c, h, w, generator=g).to(dev)
    wt = (torch.randn(4 * c, 2 * c, 3, 3, generator=g) / (2 * c * 9) ** 0.5).to(dev)
    w_in = wt[:, :c].contiguous()
    b = torch.randn(4 * c, generator=g).to(dev)
    state = (torch.tanh(torch.randn(n, c, h, w, generator=g)).to(dev), torch.randn(n, c, h, w, generator=g).to(dev))
    ch1 = K.Chain(n, c, h, w, (3, 3), 1, dev, tag="rate_zero")
    ch2 = K.Chain(n, 2 * c, h, w, (3, 3), 1, dev, tag="rate_state")
    for ch in (ch1, ch2):
        N.check(N.lib().b200_conv_tma_pack_chain(C.byref(ch.desc), N.ptr(x), c, N.ptr(ch.buf), 0, N.current_stream()))

    def pack_hidden():
        N.check(N.lib().b200_conv_tma_pack_chain(C.byref(ch2.desc), N.ptr(state[0]), c, N.ptr(ch2.buf), c,
                                                 N.current_stream()))

    def two_kernels_state_chained():
        pack_hidden()
        return K.convlstm_cell(K.conv2d(ch2, wt, b, pad=1), state[1])

    K.set_conv_precision("tc")
    variants = {
        "zero_chained_fused": lambda: K.convlstm(ch1, w_in, b),
        "zero_chained_conv_cell": lambda: K.convlstm_zero_state(K.conv2d(ch1, w_in, b, pad=1)),
        "zero_plain_fused": lambda: K.convlstm(x, w_in, b),
        "zero_plain_conv_cell": lambda: K.convlstm_zero_state(K.conv2d(x, w_in, b, pad=1)),
        "state_chained_fused": lambda: K.convlstm(ch2, wt, b, state),
        "state_chained_conv_cell": two_kernels_state_chained,
        "state_plain_fused": lambda: K.convlstm(x, wt, b, state),
        "state_plain_conv_cell": lambda: K.convlstm_cell(K.conv2d(torch.cat((x, state[0]), 1), wt, b, pad=1), state[1]),
    }
    for name, fn in variants.items():
        med, best = _time(fn, args.reps, args.warmup)
        print(json.dumps({"variant": name, "gates_hw": [h, w], "C": c, "median_ms": round(med, 4),
                          "min_ms": round(best, 4), "gpu": torch.cuda.get_device_name()}))


if __name__ == "__main__":
    main()
