#!/usr/bin/env python
"""RAFT's two correlation paths side by side at 1920 x 1080 and 3840 x 2160: the all-pairs pyramid (CorrBlock) and the
on-the-fly correlation (AlternateCorrBlock), on synthetic frame pairs with random RAFT weights.

For each frame size and each path that fits in the device's memory it prints
  * correlation only: one build + 20 lookups (CUDA events, median of 5 repetitions),
  * RAFT.forward_both with 20 refinement iterations (mixed precision, captured refinement graph; median of 3 after a
    warm-up call),
  * torch.cuda.max_memory_allocated of each run,
and the card's name and power limit.  `bench.py --workload raft` times the all-pairs path at 1080p; this adds 4K.

    python tools/raft_corr_rate.py [--sizes 1080p,4k] [--out FILE.json]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "all-in-one-deflicker_b200"))
from b200 import _native as N  # noqa: E402
from src.models.stage_1.core.corr import AlternateCorrBlock, CorrBlock  # noqa: E402
from src.models.stage_1.core.raft import RAFT  # noqa: E402
from src.models.stage_1.core.utils.utils import coords_grid  # noqa: E402

SIZES = {"1080p": (1080, 1920), "4k": (2160, 3840)}
LOOKUPS = 20


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return q or f"{torch.cuda.get_device_name(0)}, power limit unknown"


def events_ms(fn, reps):
    times = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1))
    return sorted(times)[len(times) // 2]


def fits(block, h8, w8):
    if block is AlternateCorrBlock:
        return True
    return int(N.lib().b200_corr_pyramid_floats(h8, w8)) * 4 < torch.cuda.get_device_properties(0).total_memory // 2


def corr_only(block, h8, w8):
    g = torch.Generator(device="cuda").manual_seed(0)
    f1 = torch.randn(1, 256, h8, w8, device="cuda", generator=g)
    f2 = torch.randn(1, 256, h8, w8, device="cuda", generator=g)
    # a smooth flow of a few pixels, as the refinement sees it
    ys = torch.linspace(0, 6.28, h8, device="cuda").view(h8, 1)
    xs = torch.linspace(0, 6.28, w8, device="cuda").view(1, w8)
    coords = coords_grid(1, h8, w8).cuda()
    coords[0, 0] += 3 * torch.sin(ys + xs)
    coords[0, 1] += 2 * torch.cos(xs - ys)
    coords = coords.contiguous()

    def run():
        blk = block(f1, f2)
        for _ in range(LOOKUPS):
            blk(coords)

    run()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    ms = events_ms(run, 5)
    return ms, torch.cuda.max_memory_allocated()


def forward_both(alternate, H, W):
    torch.manual_seed(0)
    model = RAFT(argparse.Namespace(small=False, mixed_precision=True, alternate_corr=alternate)).cuda().eval()
    g = torch.Generator().manual_seed(1)
    im1 = (torch.rand(1, 3, H, W, generator=g) * 255).cuda()
    im2 = torch.roll(im1, shifts=(2, -3), dims=(2, 3))
    model.forward_both(im1, im2, iters=20)             # captures the refinement graph
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    ms = events_ms(lambda: model.forward_both(im1, im2, iters=20), 3)
    peak = torch.cuda.max_memory_allocated()
    del model
    return ms, peak


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1080p,4k")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this measurement needs a CUDA device"
    torch.cuda.set_device(0)
    rows = []
    for name in args.sizes.split(","):
        H, W = SIZES[name]
        h8, w8 = H // 8, W // 8
        for label, block in (("all-pairs", CorrBlock), ("on-the-fly", AlternateCorrBlock)):
            row = {"frames": f"{W}x{H}", "features": f"{w8}x{h8}", "path": label}
            if not fits(block, h8, w8):
                gb = int(N.lib().b200_corr_pyramid_floats(h8, w8)) * 4 / 1e9
                row.update(note=f"does not fit: pyramid {gb:.1f} GB")
            else:
                torch.cuda.empty_cache()
                ms, peak = corr_only(block, h8, w8)
                row.update(corr_build_plus_20_lookups_ms=round(ms, 2), corr_peak_gb=round(peak / 1e9, 2))
                torch.cuda.empty_cache()
                ms, peak = forward_both(block is AlternateCorrBlock, H, W)
                row.update(forward_both_20_iters_ms=round(ms, 1), forward_both_peak_gb=round(peak / 1e9, 2))
            print(json.dumps(row), flush=True)
            rows.append(row)
    result = {"card": card(), "rows": rows}
    print(json.dumps({"card": result["card"]}))
    print("| frames | path | build + 20 lookups (ms) | peak (GB) | forward_both, 20 iters (ms) | peak (GB) |")
    print("|---|---|---|---|---|---|")
    for r in rows:
        if "note" in r:
            print(f"| {r['frames']} | {r['path']} | {r['note']} | | | |")
        else:
            print(f"| {r['frames']} | {r['path']} | {r['corr_build_plus_20_lookups_ms']} | {r['corr_peak_gb']} | "
                  f"{r['forward_both_20_iters_ms']} | {r['forward_both_peak_gb']} |")
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
