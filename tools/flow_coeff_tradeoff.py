"""The trade E_warp and fidelity expose together: the stage-1 atlas of one flickering video fitted at several
`optical_flow_coeff` values, each output scored by its warping error and by SSIM / PSNR against the clean frames.

    python tools/flow_coeff_tradeoff.py [--coeffs 5 500] [--frames 80] [--height 432] [--width 768] [--out DIR]

Writes synth.quality_set(H, W, T, seed=0) (a translating texture with a per-frame gain and offset) as 8-bit PNGs with
its exact flows and its flicker-free `clean` frames, fits it with `src/stage1_neural_atlas.py --down 1` and the shipped
config's iteration count at each coefficient, and scores the stage-1 output with
`src/evaluate_flicker.py --sequences input,atlas --fidelity --reference clean`.  Prints one JSON line with the card's
name and power limit, then one per coefficient.  Work files go to a temporary directory (or --out)."""
import argparse
import json
import os
import shutil
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from clip_seams import PKG, card, run, write_video  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--coeffs", type=float, nargs="+", default=[5.0, 500.0])
    ap.add_argument("--frames", type=int, default=80)
    ap.add_argument("--height", type=int, default=432)
    ap.add_argument("--width", type=int, default=768)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import cv2
    import torch
    if torch.cuda.device_count() == 0:
        sys.exit("no GPU: nothing measured")
    print(json.dumps({"cards": card()}), flush=True)
    sys.path.insert(0, PKG)
    from b200 import synth
    work = args.out or tempfile.mkdtemp(prefix="flow_coeff_")
    write_video(os.path.join(work, "data", "test", "q"), args.frames, args.height, args.width)
    q = synth.quality_set(args.height, args.width, args.frames, seed=0)
    os.makedirs(os.path.join(work, "clean"))
    for t in range(args.frames):
        img = np.round(np.clip(q["clean"][..., t].numpy(), 0, 1) * 255).astype(np.uint8)
        cv2.imwrite(os.path.join(work, "clean", "%05d.png" % t), cv2.cvtColor(img, cv2.COLOR_RGB2BGR))
    cfg = json.load(open(os.path.join(PKG, "src", "config", "config_flow_100.json")))
    cfg.update(maximum_number_of_frames=max(cfg["maximum_number_of_frames"], args.frames))
    pkg = os.path.join(work, "pkg")
    shutil.copytree(PKG, pkg, ignore=shutil.ignore_patterns("__pycache__"))
    env = dict(os.environ, PYTHONPATH=pkg, B200_ALLOW_RANDOM_RAFT="1")
    for coeff in args.coeffs:
        cfg.update(optical_flow_coeff=coeff)
        with open(os.path.join(pkg, "src", "config", "config_flow_100.json"), "w") as f:
            json.dump(cfg, f, indent=4)
        shutil.rmtree(os.path.join(work, "results"), ignore_errors=True)
        t0 = time.perf_counter()
        run([sys.executable, os.path.join(pkg, "src", "stage1_neural_atlas.py"), "--vid_name", "q", "--root",
             "data/test/", "--down", "1", "--no_artefacts"], work, env)
        stage1_s = time.perf_counter() - t0
        run([sys.executable, os.path.join(pkg, "src", "evaluate_flicker.py"), "--video_name", "q", "--sequences",
             "input,atlas", "--fidelity", "--reference", "clean"], work, env)
        flick = json.load(open(os.path.join(work, "results", "q", "flicker.json")))["sequences"]
        fid = json.load(open(os.path.join(work, "results", "q", "fidelity.json")))["sequences"]
        print(json.dumps({
            "optical_flow_coeff": coeff, "size": "%dx%d" % (args.width, args.height), "frames": args.frames,
            "iters": cfg["iters_num"], "stage1_s": round(stage1_s, 1),
            "E_warp": {s: flick[s]["E_warp"] for s in flick},
            "SSIM": {s: fid[s]["SSIM"] for s in fid}, "PSNR": {s: fid[s]["PSNR"] for s in fid}}), flush=True)
    if args.out is None:
        shutil.rmtree(work, ignore_errors=True)


if __name__ == "__main__":
    main()
