"""Stage 2 — neural filter (UNet) + local refinement (TransformNet) with the reference's CLI and output
folders (src/neural_filter_and_refinement.py).  Like the reference it requires a GPU."""
import argparse
import os
import random
import shutil
import sys
from glob import glob
from types import SimpleNamespace

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

import cv2          # noqa: E402
import numpy as np  # noqa: E402
import torch        # noqa: E402
from tqdm import tqdm  # noqa: E402

import src.models.network_filter as net  # noqa: E402
from src.models.network_local import TransformNet  # noqa: E402
from src.models.utils import InputPadder, load_image, save_img, tensor2img  # noqa: E402

parser = argparse.ArgumentParser()
parser.add_argument("--ckpt_filter", default="./pretrained_weights/neural_filter.pth", type=str)
parser.add_argument("--ckpt_local", default="./pretrained_weights/local_refinement_net.pth", type=str)
parser.add_argument("--fps", default=10, type=int)
parser.add_argument("--video_name", default=None, type=str)
parser.add_argument('--gpu', type=int, default=0)
# not in the reference: convolution arithmetic.  "tc" = wgmma with fp16 operands / fp32 accumulation — the same
# operand width as the TF32 cuDNN convolutions the reference runs by default; "fp32" = CUDA-core FFMA.
parser.add_argument('--conv_precision', choices=["tc", "fp32"], default="tc")


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
    frame_o1 = frame_p1 = None
    for i in tqdm(range(len(style_names))):
        content, org_size = load_image(content_names[i], device=device, resize=False)
        style, _ = load_image(style_names[i], size=org_size, device=device, resize=False)
        content, style = InputPadder(content.shape).pad(content, style)
        pred = filter_net(torch.cat([content, style], dim=1))
        if i == 0:
            frame_o2 = frame_o1 = frame_p1 = pred
        else:
            out, _ = local_net(torch.cat((pred, frame_o1, pred, frame_p1), dim=1), None)
            frame_o2 = pred + out
            frame_p1, frame_o1 = pred, frame_o2
        imgs = [cv2.resize(tensor2img(t), org_size, cv2.INTER_LINEAR) for t in (content, style, pred)]
        save_img(np.concatenate(imgs, axis=1), "{}/{:05d}.png".format(out_concat, i))
        save_img(imgs[2], "{}/{:05d}.png".format(out_filter, i))
        save_img(cv2.resize(tensor2img(frame_o2), org_size, cv2.INTER_LINEAR), "{}/{:05d}.png".format(out_final, i))
    if shutil.which("ffmpeg"):
        for d in (out_concat, out_filter, out_final):
            os.system("ffmpeg -y -r %s -i %s -crf 25 -r 12 -qscale 4  %s" % (opts.fps, os.path.join(d, "%05d.png"), d + ".mp4"))


if __name__ == "__main__":
    main(parser.parse_args())
