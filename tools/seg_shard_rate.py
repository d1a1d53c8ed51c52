"""What a frame shard of the segmentation trip costs, on ONE GPU: the trip (b200_seg_loss_grad) of the whole video
against the trip of rank 0 of an emulated N-way frame split (N = 2, 4, 8: rank 0's frame block resident, the same
global index batch, no collective), at the benchmark geometry (80 x 432 x 768, 10 000 samples, config_flow_100.json,
tensor cores).  A rank evaluates only the tiles that hold its resident samples, so its trip time should fall with its
share of the batch until launch latency dominates.  Prints one JSON line per configuration, with the card's name and
power limit.

    python tools/seg_shard_rate.py [--steps 50] [--warmup 5] [--fp32]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "all-in-one-deflicker_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

from b200 import _native as N, atlas as A, seg as SG, synth  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [s.strip() for s in q.split(",")]
    except Exception:                            # noqa: BLE001 - nvidia-smi missing: the name alone
        name, power = torch.cuda.get_device_name(), "unknown"
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--fp32", action="store_true")
    args = ap.parse_args()
    T, H, W, B = 80, 432, 768, 10000
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    prec = N.PREC_FP32 if args.fp32 else N.PREC_TC
    data = synth.throughput_set(H, W, T, seed=0)
    masks = (torch.rand(H, W, T, generator=torch.Generator().manual_seed(2)) < 0.4).float()
    g = torch.Generator().manual_seed(1)
    inds = [torch.randint(H * W * T, (B,), generator=g).to(dev) for _ in range(8)]
    name, power = card()
    whole_ms = None
    for world in (1, 2, 4, 8):
        t0, t1 = A.frame_range(0, world, T)
        vid = A.DeviceVideo.from_reference_layout(data, dev, t0, t1)
        tr = SG.SegTrainer(vid, SG.pack_mask_frames(masks, dev, t0, t1), None, precision=prec, device=dev)
        torch.manual_seed(0)
        tr.init_like_reference()
        resident = []
        for i in range(max(2, args.warmup)):           # both regimes: their job tables are built eagerly once
            tr.indices.copy_(inds[i % 8])
            tr.loss_grad(0 if i % 2 == 0 else 6000)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(args.steps):
            tr.indices.copy_(inds[i % 8])
            tr.loss_grad(0 if i < args.steps // 2 else 6000)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / args.steps
        for x in inds:
            t = x // (H * W)
            resident.append(int(((t >= t0) & (t < t1)).sum()))
        whole_ms = ms if world == 1 else whole_ms
        print(json.dumps({"shards": world, "rank": 0, "frames": [t0, t1], "mean_resident_samples": sum(resident) / len(resident),
                          "ms_per_trip": round(ms, 4), "vs_whole_video": round(ms / whole_ms, 4),
                          "precision": "tc" if prec == N.PREC_TC else "fp32", "card": name, "power_limit": power,
                          "geometry": f"{T}x{H}x{W}, {B} samples"}), flush=True)
        del tr, vid
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
