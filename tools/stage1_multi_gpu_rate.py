"""Wall time of the multi-GPU atlas script by phase — flow pre-pass, loading, pre-training, the loop, the evaluation —
at 1 / 2 / 4 / 8 GPUs of this node (counts above the node's GPUs are reported as not measured).

    python tools/stage1_multi_gpu_rate.py [--gpus 1 2 4 8] [--frames 80] [--iters 10001] [--out DIR]

Each count runs `src/stage1_neural_atlas.py --down 4 --gpus N` (under torch.distributed.run, also for N = 1) from scratch
on a seeded synthetic 1920x1080 clip with randomly initialised RAFT weights, evaluating once at the last iteration.
Prints one JSON line per count and one with the card name and power limit, read in the same run.  Work files go to a
temporary directory (or --out)."""
import argparse
import json
import os
import re
import shutil
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "all-in-one-deflicker_b200")


def write_clip(folder, T, H=1080, W=1920, seed=0):
    import cv2
    os.makedirs(folder, exist_ok=True)
    rng = np.random.RandomState(seed)
    base = cv2.GaussianBlur(rng.rand(H + 2 * T + 8, W + 4 * T + 8, 3).astype(np.float32), (0, 0), 6.0)
    base = (base - base.min()) / (base.max() - base.min())
    for t in range(T):
        crop = base[4 + t:4 + t + H, 4 + 2 * t:4 + 2 * t + W]
        flick = 1.0 + 0.15 * np.sin(1.7 * t)
        cv2.imwrite(os.path.join(folder, "%05d.png" % t), np.clip(crop * flick * 255.0, 0, 255).astype(np.uint8))


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return [line.strip() for line in r.stdout.splitlines() if line.strip()]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, nargs="+", default=[1, 2, 4, 8])
    ap.add_argument("--frames", type=int, default=80)
    ap.add_argument("--iters", type=int, default=10001)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    have = torch.cuda.device_count()
    if have == 0:
        sys.exit("no GPU: nothing measured")
    print(json.dumps({"cards": card()}), flush=True)
    work = args.out or tempfile.mkdtemp(prefix="stage1_mg_")
    clip = os.path.join(work, "data", "test", "clip")
    write_clip(clip, args.frames)
    cfg = json.load(open(os.path.join(PKG, "src", "config", "config_flow_100.json")))
    cfg.update(iters_num=args.iters, evaluate_every=max(args.iters - 1, 1))
    cfg_path = os.path.join(work, "cfg.json")
    json.dump(cfg, open(cfg_path, "w"))
    env = dict(os.environ, PYTHONPATH=PKG, B200_ALLOW_RANDOM_RAFT="1")
    for n in args.gpus:
        if n > have:
            print(json.dumps({"gpus": n, "measured": False, "reason": f"{have} GPU(s) on this node"}), flush=True)
            continue
        for d in ("clip_flow",):
            shutil.rmtree(os.path.join(work, "data", "test", d), ignore_errors=True)
        shutil.rmtree(os.path.join(work, "results"), ignore_errors=True)
        r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--standalone", "--nproc-per-node", str(n),
                            os.path.join(PKG, "src", "stage1_neural_atlas.py"), "--vid_name", "clip", "--root",
                            "data/test/", "--down", "4", "--config", cfg_path], cwd=work, env=env, capture_output=True,
                           text=True)
        m = re.search(r"stage1_phases (\{.*\})", r.stdout)
        if r.returncode != 0 or m is None:
            print(json.dumps({"gpus": n, "measured": False, "returncode": r.returncode,
                              "stderr": r.stderr[-1500:]}), flush=True)
            continue
        phases = json.loads(m.group(1))
        phases.pop("world", None)
        print(json.dumps({"gpus": n, "measured": True, "frames": args.frames, "size": "1920x1080 --down 4",
                          "iters": args.iters, "seconds": phases, "total_s": sum(phases.values())}), flush=True)
    if args.out is None:
        shutil.rmtree(work, ignore_errors=True)


if __name__ == "__main__":
    main()
