"""Rate of src/evaluate_flicker.py --fidelity at 1080p: frames per second scoring three sequences (atlas, filter and
final, 8-bit PNG frames) against the input, with the time split into frame decoding (on the loader thread, one window
ahead) and the device part (staging, copies, b200_fidelity, read-back).  Only the fidelity is scored: no flows are
read.  Writes its synthetic video to a temporary directory.

    python tools/fidelity_rate.py [--frames 33] [--json OUT]"""
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
SEQUENCES = ["atlas", "filter", "final"]


def write_video(root, T):
    rng = np.random.default_rng(0)
    base = rng.integers(0, 256, (H + 64, W + 64, 3), dtype=np.uint8)
    folders = {"input": os.path.join(root, "data", "test", "v"),
               "atlas": os.path.join(root, "results", "v", "stage_1", "output"),
               "filter": os.path.join(root, "results", "v", "neural_filter", "output"),
               "final": os.path.join(root, "results", "v", "final", "output")}
    for d in folders.values():
        os.makedirs(d)
    for t in range(T):
        frame = base[32 - t % 16:32 - t % 16 + H, 32:32 + W]
        for k, d in enumerate(folders.values()):
            cv2.imwrite(os.path.join(d, "%05d.png" % t), (frame // (k + 1)).astype(np.uint8))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=33)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    from b200.fidelity import FidelityScorer
    from src import evaluate_flicker as E
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    with tempfile.TemporaryDirectory() as root:
        write_video(root, args.frames)
        cwd = os.getcwd()
        os.chdir(root)
        try:
            scorer = FidelityScorer("cuda:0")
            E.evaluate_fidelity("v", SEQUENCES, None, scorer.score_frames)           # warm-up run, page cache filled
            scorer.device_seconds = 0.0
            stats = {"flow_load": 0.0, "decode": 0.0}
            t0 = time.perf_counter()
            _, doc = E.evaluate_fidelity("v", SEQUENCES, None, scorer.score_frames, stats=stats)
            wall = time.perf_counter() - t0
        finally:
            os.chdir(cwd)
    out = dict(gpu=gpu, resolution=[H, W], sequences=len(SEQUENCES), frames=args.frames, wall_s=wall,
               frames_per_s=args.frames / wall, decode_s=stats["decode"], device_s=scorer.device_seconds,
               SSIM={k: v["SSIM"] for k, v in doc["sequences"].items()},
               PSNR={k: v["PSNR"] for k, v in doc["sequences"].items()})
    print(json.dumps(out))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
