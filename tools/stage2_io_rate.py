#!/usr/bin/env python
"""Wall time per frame of the stage-2 script's frame loop, files to files, at 1080x1920 content with 270x480 atlas frames
(`--down 4`), seeded random weights, wgmma convolutions.  Arms, alternated in one process after a warm-up, each window
`--frames` frames long and closed by a device synchronise:

  host    the loop on the host helpers of src/models/utils.py (float64 load_image, pad, cat; four fp32 D2H copies,
          cv2.resize, clip, three PNG writes), everything inline (only with `--arms host,...`: it takes over a second
          per frame)
  parent  b200.stage2.Stage2.frame (frames packed and emitted on the device, uint8 images over the bus) with
          cv2.imwrite of the three images on three writer threads: the script's loop before the PNG encoder
  sync    Stage2.frame_png (the PNG files encoded on the device, file bytes over the bus), decode and plain file
          writes inline (the script's --sync_io)
  piped   the script's default: frame_png, the next decode and the previous writes on worker threads

and the split of `host` and `sync` by host clock (the device part ends in a synchronise).  Then the encoder alone
(b200.png.encode, CUDA events, median of `--encode_reps` launches) at 1080x5760 and 1080x1920: its bytes moved and
the achieved rate against the H100 SXM data sheet's 3.35 TB/s.  The sequence is generated in a
temporary folder from a seed; nothing else is read.  Also checks that every arm wrote the files `host` writes
when OpenCV runs its own resize code (cv2.ipp.setUseIPP(False)), and counts the bytes that differ from the files `host`
writes with the installed OpenCV's default back end.  One JSON line per arm and round, then a summary line.

    python tools/stage2_io_rate.py [--frames 50] [--rounds 2] [--arms parent,sync,piped] [--height 1080 --width 1920]"""
import argparse
import concurrent.futures as cf
import importlib.util
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time
import types

import cv2
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "all-in-one-deflicker_b200")
sys.path.insert(0, PKG)

from b200 import nn as K  # noqa: E402
from b200 import png as P  # noqa: E402
from b200.stage2 import Stage2  # noqa: E402
from src.models import utils as U  # noqa: E402
from src.models.network_filter import UNet  # noqa: E402
from src.models.network_local import TransformNet  # noqa: E402


def script_module():
    spec = importlib.util.spec_from_file_location("stage2_script", os.path.join(PKG, "src", "neural_filter_and_refinement.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def make_sequence(folder, n, h, w, down, seed=0):
    rng = np.random.default_rng(seed)
    hs, ws = h // down, w // down
    yy, xx = np.mgrid[0:hs, 0:ws].astype(np.float32)
    base = np.stack([127 + 90 * np.sin(xx / 17 + c) * np.cos(yy / 23 - c) for c in range(3)], axis=2)
    base += rng.normal(0, 12, base.shape)
    cn, an = [], []
    for d in ("content", "atlas"):
        os.makedirs(os.path.join(folder, d))
    for i in range(n):
        a = np.clip(np.roll(base, i, axis=1) + rng.normal(0, 2, base.shape), 0, 255).astype(np.uint8)
        c = cv2.resize(a, (w, h), interpolation=cv2.INTER_CUBIC).astype(np.float32) * (0.8 + 0.4 * rng.random())
        c = np.clip(c + rng.normal(0, 3, (h, w, 1)), 0, 255).astype(np.uint8)                     # flicker + grain
        cn.append(os.path.join(folder, "content", "%05d.png" % i))
        an.append(os.path.join(folder, "atlas", "%05d.png" % i))
        cv2.imwrite(cn[-1], c[:, :, ::-1], [cv2.IMWRITE_PNG_COMPRESSION, 1])
        cv2.imwrite(an[-1], a[:, :, ::-1], [cv2.IMWRITE_PNG_COMPRESSION, 1])
    return cn, an


def out_dirs(root):
    d = {k: os.path.join(root, k) for k in ("concat", "filter", "final")}
    for v in d.values():
        os.makedirs(v, exist_ok=True)
    return d


def host_loop(filter_net, local_net, cn, an, dirs, device, split):
    """The frame loop as the reference's script has it, on src/models/utils.py."""
    clock = time.perf_counter
    frame_o1 = frame_p1 = None
    for i in range(len(cn)):
        t0 = clock()
        content, org = U.load_image(cn[i], device=device, resize=False)
        style, _ = U.load_image(an[i], size=org, device=device, resize=False)
        torch.cuda.synchronize()
        t1 = clock()
        content, style = U.InputPadder(content.shape).pad(content, style)
        pred = filter_net(torch.cat([content, style], dim=1))
        if i == 0:
            frame_o2 = frame_o1 = frame_p1 = pred
        else:
            out, _ = local_net(torch.cat((pred, frame_o1, pred, frame_p1), dim=1), None)
            frame_o2 = pred + out
            frame_p1, frame_o1 = pred, frame_o2
        torch.cuda.synchronize()
        t2 = clock()
        imgs = [cv2.resize(U.tensor2img(t), org, cv2.INTER_LINEAR) for t in (content, style, pred)]
        final = cv2.resize(U.tensor2img(frame_o2), org, cv2.INTER_LINEAR)
        t3 = clock()
        U.save_img(np.concatenate(imgs, axis=1), "{}/{:05d}.png".format(dirs["concat"], i))
        U.save_img(imgs[2], "{}/{:05d}.png".format(dirs["filter"], i))
        U.save_img(final, "{}/{:05d}.png".format(dirs["final"], i))
        t4 = clock()
        for k, v in (("decode_h2d", t1 - t0), ("device", t2 - t1), ("d2h_resize", t3 - t2), ("clip_encode", t4 - t3)):
            split[k] = split.get(k, 0.0) + v * 1e3


def sync_loop(st, script, cn, an, dirs, split):
    clock = time.perf_counter
    st.reset()
    for i in range(len(cn)):
        t0 = clock()
        c, a = script._decode(cn[i]), script._decode(an[i])
        t1 = clock()
        files = st.frame_png(c, a)                                # ends in an event synchronise
        t2 = clock()
        for key, folder in dirs.items():
            script._write(files[key], "{}/{:05d}.png".format(folder, i))
        t3 = clock()
        for k, v in (("decode", t1 - t0), ("h2d_device_encode_d2h", t2 - t1), ("write", t3 - t2)):
            split[k] = split.get(k, 0.0) + v * 1e3


def parent_loop(st, script, cn, an, dirs):
    """The script's loop before the device encoder: Stage2.frame, cv2.imwrite at compression 0 on three threads."""
    write = lambda img, path: cv2.imwrite(path, img, [cv2.IMWRITE_PNG_COMPRESSION, 0])
    n = len(cn)
    st.reset()
    decoder, writers = cf.ThreadPoolExecutor(1), cf.ThreadPoolExecutor(3)
    try:
        load = lambda i: (decoder.submit(script._decode, cn[i]), decoder.submit(script._decode, an[i]))
        nxt, pending = (load(0) if n else None), []
        for i in range(n):
            content, style = (f.result() for f in nxt)
            nxt = load(i + 1) if i + 1 < n else None
            for f in pending[:-1]:
                for w in f:
                    w.result()
            pending = pending[-1:]
            imgs = st.frame(content, style)
            pending.append([writers.submit(write, imgs[key], "{}/{:05d}.png".format(folder, i))
                            for key, folder in dirs.items()])
        for f in pending:
            for w in f:
                w.result()
    finally:
        decoder.shutdown(wait=True, cancel_futures=True)
        writers.shutdown(wait=True, cancel_futures=True)


def encode_rate(h, w, reps, dev):
    """b200.png.encode of a seeded (h, w, 3) image: median ms over `reps` launches (CUDA events), bytes moved, GB/s.
    Bytes: the image read once, the filtered rows written and read back, the file written."""
    rng = np.random.default_rng(h + w)
    img = torch.from_numpy(rng.integers(0, 256, (h, w, 3), dtype=np.uint8)).to(dev)
    plan = P.plan(h, w, dev)
    ws = torch.empty(plan.workspace_bytes, dtype=torch.uint8, device=dev)
    out = torch.empty(plan.file_bytes, dtype=torch.uint8, device=dev)
    for _ in range(5):
        P.encode(img, out=out, workspace=ws)
    ms = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        P.encode(img, out=out, workspace=ws)
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    assert out.cpu().numpy().tobytes() == cv2.imencode(".png", img.cpu().numpy(), [cv2.IMWRITE_PNG_COMPRESSION, 0])[1].tobytes()
    med = statistics.median(ms)
    moved = img.numel() + 2 * plan.header.raw_bytes + plan.file_bytes
    return {"shape": [h, w], "encode_ms_median": round(med, 4), "encode_ms_min": round(min(ms), 4), "launches": reps,
            "bytes_moved": int(moved), "GB_per_s": round(moved / med / 1e6, 1),
            "share_of_3.35_TB_per_s": round(moved / med / 1e6 / 3350, 3)}


def d2h_ms(st, reps=20):
    """The uint8 result copy alone (device -> pinned), CUDA events."""
    ms = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        st._host[0].copy_(st._out, non_blocking=True)
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    return statistics.median(ms)


def files(dirs, n):
    return [open(os.path.join(v, "%05d.png" % i), "rb").read() for v in dirs.values() for i in range(n)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--down", type=int, default=4)
    ap.add_argument("--arms", default="parent,sync,piped")
    ap.add_argument("--encode_reps", type=int, default=100)
    args = ap.parse_args()
    arms = args.arms.split(",")
    assert torch.cuda.is_available(), "this measurement needs a GPU"
    dev = torch.device("cuda:0")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    K.set_conv_precision("tc")
    torch.manual_seed(0)
    unet = UNet(in_channels=6, out_channels=3, init_features=32).to(dev).eval()
    tn = TransformNet(types.SimpleNamespace(nf=32, norm="IN", model="TransformNet", blocks=5), nc_in=12, nc_out=3).to(dev).eval()
    script = script_module()
    st = Stage2(unet, tn, dev)
    n = args.frames
    with tempfile.TemporaryDirectory() as tmp, torch.no_grad():
        cn, an = make_sequence(os.path.join(tmp, "in"), n, args.height, args.width, args.down)
        dirs = {arm: out_dirs(os.path.join(tmp, arm)) for arm in arms + ["host_own"]}

        def run(arm, k, split):
            if arm == "host":
                host_loop(unet, tn, cn[:k], an[:k], dirs[arm], dev, split)
            elif arm == "parent":
                parent_loop(st, script, cn[:k], an[:k], dirs[arm])
            elif arm == "sync":
                sync_loop(st, script, cn[:k], an[:k], dirs[arm], split)
            else:
                script.run_frames(st, cn[:k], an[:k], dirs[arm])
        for arm in arms:
            run(arm, args.warmup, {})
        per_frame = {arm: [] for arm in arms}
        for r in range(args.rounds):
            for arm in arms:
                split = {}
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                run(arm, n, split)
                torch.cuda.synchronize()
                ms = (time.perf_counter() - t0) * 1e3 / n
                per_frame[arm].append(ms)
                print(json.dumps({"arm": arm, "round": r, "frames": n, "ms_per_frame": round(ms, 2),
                                  "split_ms_per_frame": {k: round(v / n, 2) for k, v in split.items()}, "gpu": card}),
                      flush=True)
        # the files: against the host loop with OpenCV's own resize code (what the kernels restate) they are equal
        k = min(n, 3)
        was = cv2.ipp.useIPP()
        cv2.ipp.setUseIPP(False)
        host_loop(unet, tn, cn[:k], an[:k], dirs["host_own"], dev, {})
        cv2.ipp.setUseIPP(was)
        for arm in arms:
            assert files(dirs[arm], k) == files(dirs["host_own"], k), "%s wrote other files than the host loop" % arm
        extra = {}
        if "host" in arms:
            a = np.concatenate([cv2.imread(os.path.join(v, "%05d.png" % i)).ravel() for v in dirs["host"].values() for i in range(k)])
            b = np.concatenate([cv2.imread(os.path.join(v, "%05d.png" % i)).ravel() for v in dirs[arms[-1]].values() for i in range(k)])
            diff = a.astype(np.int16) - b
            extra = {"installed_opencv_uses_ipp": bool(was), "bytes_differing_from_installed_default": float((diff != 0).mean()),
                     "max_level_difference": int(np.abs(diff).max())}
        for h, w in ((1080, 5760), (1080, 1920)):
            print(json.dumps(dict(encode_rate(h, w, args.encode_reps, dev), gpu=card)), flush=True)
        print(json.dumps(dict({"summary": True, "geometry": [args.height, args.width, args.down], "frames_per_window": n,
                               "ms_per_frame_median": {k_: round(statistics.median(v), 2) for k_, v in per_frame.items()},
                               "result_d2h_ms": round(d2h_ms(st), 3), "files_equal_opencv_own_code": True, "gpu": card},
                              **extra)))


if __name__ == "__main__":
    main()
