"""Rate of src/evaluate_flicker.py at 1080p: pairs per second scoring four sequences (8-bit PNG frames, flows at the
frame size), with the time split into flow loading and frame decoding (on the loader thread, one window ahead) and the
device part (staging, copies, b200_warp_error, read-back).  Writes its synthetic video to a temporary directory.

    python tools/flicker_rate.py [--frames 33] [--json OUT]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "all-in-one-deflicker_b200")
sys.path[:0] = [PKG]

import cv2  # noqa: E402
import numpy as np  # noqa: E402
import torch  # noqa: E402

H, W = 1080, 1920


def write_video(root, T):
    rng = np.random.default_rng(0)
    base = rng.integers(0, 256, (H + 64, W + 64, 3), dtype=np.uint8)
    folders = {"input": os.path.join(root, "data", "test", "v"),
               "atlas": os.path.join(root, "results", "v", "stage_1", "output"),
               "filter": os.path.join(root, "results", "v", "neural_filter", "output"),
               "final": os.path.join(root, "results", "v", "final", "output")}
    for d in folders.values():
        os.makedirs(d)
    flow_dir = folders["input"] + "_flow"
    os.makedirs(flow_dir)
    for t in range(T):
        frame = base[32 - t % 16:32 - t % 16 + H, 32:32 + W]
        for k, d in enumerate(folders.values()):
            cv2.imwrite(os.path.join(d, "%05d.png" % t), (frame // (k + 1)).astype(np.uint8))
    F = np.zeros((H, W, 2), np.float32)
    F[..., 1] = 1.0
    for t in range(T - 1):
        a, b = "%05d.png" % t, "%05d.png" % (t + 1)
        np.save(os.path.join(flow_dir, "%s_%s.npy" % (a, b)), F)
        np.save(os.path.join(flow_dir, "%s_%s.npy" % (b, a)), -F)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=33)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    from b200.flicker import FlickerScorer
    from src import evaluate_flicker as E
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    with tempfile.TemporaryDirectory() as root:
        write_video(root, args.frames)
        cwd = os.getcwd()
        os.chdir(root)
        try:
            scorer = FlickerScorer("cuda:0")
            E.evaluate("v", list(E.SEQUENCES), scorer.score_window)             # warm-up run, page cache filled
            scorer.device_seconds = 0.0
            stats = {"flow_load": 0.0, "decode": 0.0}
            t0 = time.perf_counter()
            doc = E.evaluate("v", list(E.SEQUENCES), scorer.score_window, stats=stats)
            wall = time.perf_counter() - t0
        finally:
            os.chdir(cwd)
    pairs = args.frames - 1
    out = dict(gpu=gpu, resolution=[H, W], sequences=4, pairs=pairs, wall_s=wall, pairs_per_s=pairs / wall,
               flow_load_s=stats["flow_load"], decode_s=stats["decode"], device_s=scorer.device_seconds,
               E_warp={k: v["E_warp"] for k, v in doc["sequences"].items()})
    print(json.dumps(out))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
