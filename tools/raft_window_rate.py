#!/usr/bin/env python
"""Where the RAFT flow pre-pass spends its time, and the windowed pre-pass against the per-pair one.

    python tools/raft_window_rate.py [--frames 80] [--rounds 2] [--json out.json]

1. The per-pair loop (decode both files of the pair, one compute_flow_both call, two np.save calls) on a seeded
   1920x1080 clip, split into decode, host-to-device copy, encoders (fnet on both frames, cnet per direction),
   correlation build, refinement (20 iterations per direction, captured graph), device-to-host copy and np.save.  Each
   phase ends in a device synchronise, so the phases add up to more than the pipelined loop takes.
2. The whole pre-pass at 640x360 and 1920x1080: src/preprocess_optical_flow.preprocess (windows) against the per-pair
   loop, alternated, with pairs/s and the peak allocated device memory of each.
Random RAFT weights (the arithmetic, not the flow quality, sets the time).  The card's name and power limit are read
in the same process."""
import argparse
import gc
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time
from pathlib import Path

import cv2
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "all-in-one-deflicker_b200"))
from src import preprocess_optical_flow as PP  # noqa: E402
from src.models.stage_1 import raft_wrapper as RW  # noqa: E402
from src.models.stage_1.core.raft import corr_block_class  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def make_clip(root, T, H, W, seed=7):
    vid = Path(root) / f"clip_{W}x{H}"
    vid.mkdir()
    g = np.random.default_rng(seed)
    base = cv2.resize((g.random((H // 8, W // 8, 3)) * 255).astype(np.float32), (W + 4 * T, H + 2 * T),
                      interpolation=cv2.INTER_CUBIC)
    for t in range(T):
        frame = np.clip(base[t:t + H, 2 * t:2 * t + W] + g.normal(0, 2, (H, W, 3)), 0, 255).astype(np.uint8)
        cv2.imwrite(str(vid / f"{t:05d}.png"), frame)
    return vid


def sync_time(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t


def split_per_pair(vid, out_dir):
    """Phase times of the per-pair loop, summed over the pairs."""
    torch.manual_seed(0)
    raft = RW.RAFTWrapper(model_path=None, max_long_edge=2000)
    model = raft.model
    frames = sorted(vid.glob("*.png"))
    out_dir.mkdir(exist_ok=True)
    t = dict(decode=0.0, h2d=0.0, encoders=0.0, corr_build=0.0, refinement=0.0, d2h=0.0, np_save=0.0)
    iters = RW.REFINEMENT_ITERS
    for a, b in zip(frames, frames[1:]):
        t0 = time.perf_counter()
        cpu = torch.stack([raft.load_image(str(a)), raft.load_image(str(b))])
        t["decode"] += time.perf_counter() - t0
        pair, dt = sync_time(lambda: RW.InputPadder(cpu.shape).pad(cpu.to(RW.device))[0])
        t["h2d"] += dt
        x = (2 * (pair / 255.0) - 1.0).contiguous()

        def encoders():
            with model._autocast():
                f1, f2 = model.fnet([x[0:1], x[1:2]])
                return f1, f2, model.cnet(x[0:1]), model.cnet(x[1:2])
        (f1, f2, c1, c2), dt = sync_time(encoders)
        t["encoders"] += dt
        block = corr_block_class(model.args, f1.shape[-2], f1.shape[-1],
                                 torch.cuda.get_device_properties(f1.device).total_memory)
        _, dt = sync_time(lambda: (block(f1.float(), f2.float()), block(f2.float(), f1.float())))
        t["corr_build"] += dt
        # _refine builds the correlation state again into the graph's buffer, then replays the captured loop
        (r12, r21), dt = sync_time(lambda: (model._refine(f1, f2, c1, iters, None, True),
                                            model._refine(f2, f1, c2, iters, None, True)))
        t["refinement"] += dt
        (h12, h21), dt = sync_time(lambda: (RW._to_hw2(r12[1]), RW._to_hw2(r21[1])))
        t["d2h"] += dt
        t0 = time.perf_counter()
        np.save(out_dir / f"{a.name}_{b.name}.npy", h12)
        np.save(out_dir / f"{b.name}_{a.name}.npy", h21)
        t["np_save"] += time.perf_counter() - t0
    # the first pair also captures the graphs; its refinement is in the sum
    t["refinement"] -= t["corr_build"]            # the build inside _refine, measured on its own above
    n = len(frames) - 1
    return {k: v / n for k, v in t.items()}, n


def per_pair(vid, flow_dir):
    """The per-pair pre-pass: both files of every pair decoded, one compute_flow_both call, two np.save calls."""
    torch.manual_seed(0)
    raft = RW.RAFTWrapper(model_path=None, max_long_edge=2000)
    frames = sorted(vid.glob("*.png"))
    flow_dir.mkdir(exist_ok=True)
    for a, b in zip(frames, frames[1:]):
        fwd, bwd = raft.compute_flow_both(*raft.load_images(str(a), str(b)))
        np.save(flow_dir / f"{a.name}_{b.name}.npy", fwd)
        np.save(flow_dir / f"{b.name}_{a.name}.npy", bwd)


def windowed(vid, flow_dir):
    torch.manual_seed(0)
    PP.preprocess(argparse.Namespace(vid_path=vid, max_long_edge=2000))


def timed_run(fn, vid):
    flow_dir = vid.parent / (vid.name + "_flow")
    shutil.rmtree(flow_dir, ignore_errors=True)
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    fn(vid, flow_dir)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    peak = (torch.cuda.max_memory_allocated() - base) / 2 ** 30
    files = {p.name: p.read_bytes() for p in flow_dir.glob("*.npy")}
    return dt, peak, files


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=80)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    json_path = os.path.abspath(args.json) if args.json else None
    assert torch.cuda.is_available(), "this tool measures on the GPU"
    os.environ["B200_ALLOW_RANDOM_RAFT"] = "1"
    result = {"card": card(), "frames": args.frames}
    print("card:", result["card"])
    with tempfile.TemporaryDirectory() as tmp:
        os.chdir(tmp)                            # no pretrained_weights/ here: random weights, on purpose
        vid = make_clip(tmp, args.frames, 1080, 1920)
        phases, n = split_per_pair(vid, Path(tmp) / "split_out")
        result["per_pair_phases_s"] = phases
        print(f"per-pair loop at 1920x1080, {n} pairs, seconds per pair: "
              + ", ".join(f"{k} {v:.4f}" for k, v in phases.items()) + f"; sum {sum(phases.values()):.4f}")
        shutil.rmtree(Path(tmp) / "split_out")
        gc.collect()
        torch.cuda.empty_cache()
        for H, W in ((360, 640), (1080, 1920)):
            v = vid if (H, W) == (1080, 1920) else make_clip(tmp, args.frames, H, W)
            H8, W8 = (H + 7) // 8, (W + 7) // 8
            free, total = torch.cuda.mem_get_info()
            k = PP.window_pairs(H8, W8, args.frames - 1, free, total)
            runs = {"per_pair": [], "window": []}
            ref = None
            for r in range(args.rounds):
                order = ("per_pair", "window") if r % 2 == 0 else ("window", "per_pair")
                for name in order:
                    dt, peak, files = timed_run(per_pair if name == "per_pair" else windowed, v)
                    if ref is None:
                        ref = files
                    assert files == ref, f"{name} wrote different files"
                    runs[name].append((dt, peak))
                    print(f"{W}x{H} {name} round {r}: {dt:.2f} s, {(args.frames - 1) / dt:.2f} pairs/s, "
                          f"peak {peak:.2f} GB")
            entry = {"window_pairs": k}
            for name, rs in runs.items():
                best = min(x[0] for x in rs)
                entry[name] = {"seconds": [x[0] for x in rs], "pairs_per_s_best": (args.frames - 1) / best,
                               "peak_gb": max(x[1] for x in rs)}
            entry["speedup_best"] = entry["window"]["pairs_per_s_best"] / entry["per_pair"]["pairs_per_s_best"]
            result[f"{W}x{H}"] = entry
            print(f"{W}x{H}: window of {k} pairs; per-pair {entry['per_pair']['pairs_per_s_best']:.2f} pairs/s, "
                  f"window {entry['window']['pairs_per_s_best']:.2f} pairs/s ({entry['speedup_best']:.2f}x), "
                  f"files byte-identical")
            gc.collect()
            torch.cuda.empty_cache()
    result["card_after"] = card()
    line = json.dumps(result)
    print(line)
    if json_path:
        with open(json_path, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
