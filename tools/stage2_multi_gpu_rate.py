"""Frames per second of the stage-2 script's frame loop at 1 / 2 / 4 / 8 GPUs of this node (counts above the node's
GPUs are reported as not measured).

    python tools/stage2_multi_gpu_rate.py [--gpus 1 2 4 8] [--frames 48] [--out DIR]

Each count runs `src/neural_filter_and_refinement.py` under torch.distributed.run (also for N = 1) on a seeded
synthetic clip of 1920x1080 content frames and 480x270 stage-1 frames, with randomly initialised UNet and
TransformNet weights.  The rate is the frame count over the loop's wall time as rank 0 prints it (`stage2_loop`:
from a barrier before the loop to a device synchronise and a barrier after it), so model loading and the videos are
not in it.  Prints one JSON line per count and one with the card name and power limit, read in the same run.  Work
files go to a temporary directory (or --out)."""
import argparse
import json
import os
import re
import shutil
import subprocess
import sys
import tempfile
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "all-in-one-deflicker_b200")
sys.path.insert(0, os.path.join(ROOT, "tools"))

from stage1_multi_gpu_rate import card, write_clip  # noqa: E402


def write_inputs(work, T, seed=0):
    """data/test/clip (1080p content), results/clip/stage_1/output (270x480 atlas frames), pretrained_weights/."""
    import cv2
    import torch
    sys.path.insert(0, PKG)
    from src.models.network_filter import UNet
    from src.models.network_local import TransformNet
    content = os.path.join(work, "data", "test", "clip")
    write_clip(content, T, seed=seed)
    atlas = os.path.join(work, "results", "clip", "stage_1", "output")
    os.makedirs(atlas, exist_ok=True)
    for name in sorted(os.listdir(content)):
        img = cv2.imread(os.path.join(content, name))
        cv2.imwrite(os.path.join(atlas, name), cv2.resize(img, (480, 270), interpolation=cv2.INTER_AREA))
    weights = os.path.join(work, "pretrained_weights")
    os.makedirs(weights, exist_ok=True)
    torch.manual_seed(seed)
    torch.save(UNet(in_channels=6, out_channels=3, init_features=32).state_dict(), os.path.join(weights, "neural_filter.pth"))
    tn = TransformNet(types.SimpleNamespace(nf=32, norm="IN", model="TransformNet", blocks=5), nc_in=12, nc_out=3)
    torch.save(tn.state_dict(), os.path.join(weights, "local_refinement_net.pth"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, nargs="+", default=[1, 2, 4, 8])
    ap.add_argument("--frames", type=int, default=48)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    have = torch.cuda.device_count()
    if have == 0:
        sys.exit("no GPU: nothing measured")
    print(json.dumps({"cards": card()}), flush=True)
    work = args.out or tempfile.mkdtemp(prefix="stage2_mg_")
    write_inputs(work, args.frames)
    env = dict(os.environ, PYTHONPATH=PKG)
    for k in ("WORLD_SIZE", "RANK", "LOCAL_RANK"):
        env.pop(k, None)
    for n in args.gpus:
        if n > have:
            print(json.dumps({"gpus": n, "measured": False, "reason": f"{have} GPU(s) on this node"}), flush=True)
            continue
        for d in ("neural_filter", "final"):
            shutil.rmtree(os.path.join(work, "results", "clip", d), ignore_errors=True)
        r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--standalone", "--nproc-per-node", str(n),
                            os.path.join(PKG, "src", "neural_filter_and_refinement.py"), "--video_name", "clip"],
                           cwd=work, env=env, capture_output=True, text=True)
        m = re.search(r"stage2_loop (\{.*\})", r.stdout)
        if r.returncode != 0 or m is None:
            print(json.dumps({"gpus": n, "measured": False, "returncode": r.returncode,
                              "stderr": r.stderr[-1500:]}), flush=True)
            continue
        loop = json.loads(m.group(1))
        print(json.dumps({"gpus": n, "measured": True, "frames": loop["frames"], "size": "1920x1080, atlas 480x270",
                          "loop_s": loop["seconds"], "frames_per_s": loop["frames"] / loop["seconds"]}), flush=True)
    if args.out is None:
        shutil.rmtree(work, ignore_errors=True)


if __name__ == "__main__":
    main()
