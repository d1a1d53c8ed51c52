"""Stage 2 — neural filter (UNet) + local refinement (TransformNet) with the reference's CLI and output
folders (src/neural_filter_and_refinement.py).  Like the reference it requires a GPU.

The frames stay on the device (b200.stage2.Stage2), and so does the PNG encoding of the three output images
(Stage2.frame_png: the files cv2.imwrite writes at compression 0, byte for byte): the host decodes the 8-bit input PNGs
and writes finished files, the next frame's decode on one thread and the previous frame's three writes on a small pool
while the current frame is on the GPU."""
import argparse
import concurrent.futures as cf
import os
import random
import shutil
import sys
from glob import glob
from types import SimpleNamespace

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

import numpy as np  # noqa: E402
import torch        # noqa: E402
from tqdm import tqdm  # noqa: E402

import src.models.network_filter as net  # noqa: E402
from src.models.network_local import TransformNet  # noqa: E402
from PIL import Image  # noqa: E402

parser = argparse.ArgumentParser()
parser.add_argument("--ckpt_filter", default="./pretrained_weights/neural_filter.pth", type=str)
parser.add_argument("--ckpt_local", default="./pretrained_weights/local_refinement_net.pth", type=str)
parser.add_argument("--fps", default=10, type=int)
parser.add_argument("--video_name", default=None, type=str)
parser.add_argument('--gpu', type=int, default=0)
# not in the reference: convolution arithmetic.  "tc" = wgmma with fp16 operands / fp32 accumulation — the same
# operand width as the TF32 cuDNN convolutions the reference runs by default; "fp32" = CUDA-core FFMA.
parser.add_argument('--conv_precision', choices=["tc", "fp32"], default="tc")
# not in the reference: decode and write inline instead of on worker threads (debugging; the comparison arm of
# tools/stage2_io_rate.py).  The files are the same either way.
parser.add_argument('--sync_io', action="store_true")


def _decode(path):
    return np.array(Image.open(path))


def _write(data, path):
    with open(path, "wb") as f:
        f.write(data)


def run_frames(stage2, content_names, style_names, out_dirs, sync_io=False, progress=lambda it: it):
    """The frame loop: out_dirs = {"concat", "filter", "final"} -> folder.  Pipelined unless sync_io: frame i + 1 is
    decoded and frame i - 1 written while frame i is on the GPU.  A frame's files are views of a buffer Stage2 reuses
    two calls later, so frame i's writes are awaited before frame i + 2 starts.  Every thread is joined on return and
    on any exception."""
    n = len(content_names)
    stage2.reset()
    if sync_io:
        for i in progress(range(n)):
            imgs = stage2.frame_png(_decode(content_names[i]), _decode(style_names[i]))
            for key, folder in out_dirs.items():
                _write(imgs[key], "{}/{:05d}.png".format(folder, i))
        return
    decoder, writers = cf.ThreadPoolExecutor(1), cf.ThreadPoolExecutor(3)
    try:
        load = lambda i: (decoder.submit(_decode, content_names[i]), decoder.submit(_decode, style_names[i]))
        nxt, pending = (load(0) if n else None), []
        for i in progress(range(n)):
            content, style = (f.result() for f in nxt)
            nxt = load(i + 1) if i + 1 < n else None
            for f in pending[:-1]:                               # frame i - 2: its buffer is about to be reused
                for w in f:
                    w.result()
            pending = pending[-1:]
            imgs = stage2.frame_png(content, style)
            pending.append([writers.submit(_write, imgs[key], "{}/{:05d}.png".format(folder, i))
                            for key, folder in out_dirs.items()])
        for f in pending:
            for w in f:
                w.result()
    finally:
        decoder.shutdown(wait=True, cancel_futures=True)
        writers.shutdown(wait=True, cancel_futures=True)


def main(opts):
    seed = 2023
    np.random.seed(seed); torch.manual_seed(seed); random.seed(seed)
    if not torch.cuda.is_available():
        raise Exception("No GPU found, run with cpu")
    device = torch.device("cuda:{}".format(opts.gpu))
    from b200 import nn as K
    K.set_conv_precision(opts.conv_precision)
    filter_net = net.UNet(in_channels=6, out_channels=3, init_features=32)
    filter_net.load_state_dict(torch.load(opts.ckpt_filter, map_location="cpu"))
    filter_net.to(device).eval()
    local_net = TransformNet(SimpleNamespace(nf=32, norm='IN', model='TransformNet', blocks=5), nc_in=12, nc_out=3)
    local_net.load_state_dict(torch.load(opts.ckpt_local, map_location="cpu"))
    local_net.to(device).eval()

    style_names = sorted(glob("./results/{}/stage_1/output/*".format(opts.video_name)))
    content_names = sorted(glob("./data/test/{}/*".format(opts.video_name)))
    assert len(style_names) == len(content_names), "the number of style frames is different from the number of content frames"
    out_concat = "./results/{}/neural_filter/concat".format(opts.video_name)
    out_filter = "./results/{}/neural_filter/output".format(opts.video_name)
    out_final = os.path.join("results", opts.video_name, "final", "output")
    for d in (out_concat, out_filter, out_final):
        os.makedirs(d, exist_ok=True)
    from b200.stage2 import Stage2
    run_frames(Stage2(filter_net, local_net, device), content_names, style_names,
               {"concat": out_concat, "filter": out_filter, "final": out_final}, sync_io=opts.sync_io, progress=tqdm)
    if shutil.which("ffmpeg"):
        for d in (out_concat, out_filter, out_final):
            os.system("ffmpeg -y -r %s -i %s -crf 25 -r 12 -qscale 4  %s" % (opts.fps, os.path.join(d, "%05d.png"), d + ".mp4"))


if __name__ == "__main__":
    main(parser.parse_args())
