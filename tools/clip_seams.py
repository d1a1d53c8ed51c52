"""The seam between clip atlases, without and with a cross-fade over overlapping frames (`--clips --clip_overlap V`).

    python tools/clip_seams.py [--frames 120] [--max_frames 50] [--overlaps 0 8] [--height 270] [--width 480] [--out DIR] [--fidelity]

Writes a seeded flickering synthetic video (b200.synth.quality_set: a translating texture with a per-frame gain and
offset) with its exact flows, fits it with `src/stage1_neural_atlas.py --clips` at each overlap V with the shipped
config's iteration count (maximum_number_of_frames set to --max_frames), and scores the stage-1 output with
`src/evaluate_flicker.py --clips --clip_overlap V` (with --fidelity, also the atlas output's SSIM and PSNR against the
input, seam and interior frames apart).  Prints one JSON line per V: the plan, E_boundary and E_interior of
the input and of the atlas output, the seam pairs' E(t), the wall time of the whole stage-1 run and of the stitch; and
one line with the card's name and power limit, read in the same run.  Work files go to a temporary directory (or
--out)."""
import argparse
import json
import os
import re
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "all-in-one-deflicker_b200")
sys.path.insert(0, PKG)


def write_video(folder, T, H, W, seed=0):
    """quality_set's flickering frames as 8-bit PNGs and its exact flows where the pre-pass writes RAFT's."""
    import cv2
    from b200 import synth
    q = synth.quality_set(H, W, T, seed=seed)
    os.makedirs(folder)
    os.makedirs(folder + "_flow")
    for t in range(T):
        img = np.round(np.clip(q["frames"][..., t].numpy(), 0, 1) * 255).astype(np.uint8)
        cv2.imwrite(os.path.join(folder, "%05d.png" % t), cv2.cvtColor(img, cv2.COLOR_RGB2BGR))
    for t in range(T - 1):
        a, b = "%05d.png" % t, "%05d.png" % (t + 1)
        np.save(os.path.join(folder + "_flow", "%s_%s.npy" % (a, b)), q["flow_fwd"][:, :, :, t, 0].numpy())
        np.save(os.path.join(folder + "_flow", "%s_%s.npy" % (b, a)), q["flow_bwd"][:, :, :, t + 1, 0].numpy())


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return [line.strip() for line in r.stdout.splitlines() if line.strip()]


def run(cmd, cwd, env):
    r = subprocess.run(cmd, cwd=cwd, env=env, capture_output=True, text=True)
    if r.returncode != 0:
        sys.exit("failed: %s\n%s\n%s" % (" ".join(cmd), r.stdout[-2000:], r.stderr[-4000:]))
    return r.stdout


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=120)
    ap.add_argument("--max_frames", type=int, default=50)
    ap.add_argument("--overlaps", type=int, nargs="+", default=[0, 8])
    ap.add_argument("--height", type=int, default=270)
    ap.add_argument("--width", type=int, default=480)
    ap.add_argument("--out", default=None)
    ap.add_argument("--fidelity", action="store_true",
                    help="also score the atlas output's SSIM and PSNR against the input, seam and interior frames apart")
    args = ap.parse_args()
    import torch
    if torch.cuda.device_count() == 0:
        sys.exit("no GPU: nothing measured")
    print(json.dumps({"cards": card()}), flush=True)
    from b200 import atlas as A
    work = args.out or tempfile.mkdtemp(prefix="clip_seams_")
    write_video(os.path.join(work, "data", "test", "seams"), args.frames, args.height, args.width)
    cfg = json.load(open(os.path.join(PKG, "src", "config", "config_flow_100.json")))
    cfg.update(maximum_number_of_frames=args.max_frames)
    # evaluate_flicker reads maximum_number_of_frames from the package's config: run both from a copy that ships this one
    pkg = os.path.join(work, "pkg")
    shutil.copytree(PKG, pkg, ignore=shutil.ignore_patterns("__pycache__"))
    with open(os.path.join(pkg, "src", "config", "config_flow_100.json"), "w") as f:
        json.dump(cfg, f, indent=4)
    env = dict(os.environ, PYTHONPATH=pkg, B200_ALLOW_RANDOM_RAFT="1")
    for V in args.overlaps:
        shutil.rmtree(os.path.join(work, "results"), ignore_errors=True)
        extra = ["--clip_overlap", str(V)] if V > 0 else []
        t0 = time.perf_counter()
        out = run([sys.executable, os.path.join(pkg, "src", "stage1_neural_atlas.py"), "--vid_name", "seams", "--root",
                   "data/test/", "--down", "1", "--no_artefacts", "--clips"] + extra, work, env)
        stage1_s = time.perf_counter() - t0
        m = re.search(r"stitch: rank 0 wrote (\d+) frames of \d+ seams in ([0-9.]+) s", out)
        run([sys.executable, os.path.join(pkg, "src", "evaluate_flicker.py"), "--video_name", "seams", "--sequences",
             "input,atlas", "--clips"] + extra + (["--fidelity"] if args.fidelity else []), work, env)
        fid = {}
        if args.fidelity:
            f = json.load(open(os.path.join(work, "results", "seams", "fidelity.json")))["sequences"]["atlas"]
            fid = {k: f[k] for k in ("SSIM", "PSNR", "SSIM_seam", "SSIM_interior", "PSNR_seam", "PSNR_interior")}
        doc = json.load(open(os.path.join(work, "results", "seams", "flicker.json")))
        seqs = doc["sequences"]
        pairs = doc["clips"]["boundary_pairs"]
        print(json.dumps({
            "overlap": V, "frames": args.frames, "size": "%dx%d" % (args.width, args.height),
            "max_frames": args.max_frames, "iters": cfg["iters_num"], "plan": doc["clips"]["plan"],
            "seams": [list(s) for s in A.clip_seams(A.clip_plan(args.frames, args.max_frames, V))],
            "E_boundary": {s: seqs[s]["E_boundary"] for s in seqs},
            "E_interior": {s: seqs[s]["E_interior"] for s in seqs},
            "atlas_seam_pairs": {t: seqs["atlas"]["per_pair"][t]["E"] for t in pairs},
            "stage1_s": round(stage1_s, 1),
            "stitched_frames": int(m.group(1)) if m else 0, "stitch_s": float(m.group(2)) if m else None,
            **({"atlas_fidelity": fid} if fid else {})}), flush=True)
    if args.out is None:
        shutil.rmtree(work, ignore_errors=True)


if __name__ == "__main__":
    main()
