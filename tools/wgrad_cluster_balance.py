"""Spread of per-cluster busy time of the weight-gradient kernel at the benchmark configuration, on one GPU.

    python tools/wgrad_cluster_balance.py

tc_wgrad_kernel runs in clusters of two CTAs, and CTAs 2c and 2c + 1 form cluster c.  The two CTAs wait for each
other at every ring slot, so a cluster's time is the later of its two CTAs' (b200_debug_wgrad: per-CTA cycles of the
last launch).  Prints one JSON line per regime (with / without the global rigidity term) with the card's name and
power limit: the number of clusters, their mean cycles, and the least and largest cluster time over that mean.
"""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "all-in-one-deflicker_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)
from b200 import _native as N, atlas as A, synth  # noqa: E402

H, W, T, B = 432, 768, 80, 10000


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    assert torch.cuda.is_available(), "needs a CUDA device"
    data = synth.throughput_set(H, W, T, seed=0)
    vid = A.DeviceVideo.from_reference_layout(data, "cuda")
    tr = A.AtlasTrainer(vid, {"samples_batch": B}, precision=N.PREC_TC, device="cuda")
    torch.manual_seed(0); tr.init_like_reference()
    inds = torch.randint(H * W * T, (B,), generator=torch.Generator().manual_seed(1)).cuda()
    for wg in (True, False):
        for _ in range(3):
            tr.indices.copy_(inds); tr.loss_grad(wg)
        torch.cuda.synchronize()
        cyc = (C.c_longlong * 256)(); shp = (C.c_int32 * 768)()
        n = N.lib().b200_debug_wgrad(cyc, shp, 256)
        assert n > 0 and n % 2 == 0, n
        c = np.array(cyc[:n], dtype=np.float64)
        per_cluster = np.maximum(c[0::2], c[1::2])
        print(json.dumps({"regime": "with_global" if wg else "without", "card": card(), "clusters": int(per_cluster.size),
                          "mean_cycles": int(per_cluster.mean()),
                          "min_rel": round(float(per_cluster.min() / per_cluster.mean()), 3),
                          "max_rel": round(float(per_cluster.max() / per_cluster.mean()), 3)}))


if __name__ == "__main__":
    main()
