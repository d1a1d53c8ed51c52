"""Stage 2 — neural filter (UNet) + local refinement (TransformNet) with the reference's CLI and output
folders (src/neural_filter_and_refinement.py).  Like the reference it requires a GPU.

The frames stay on the device (b200.stage2.Stage2), and so does the PNG encoding of the three output images
(Stage2.frame_png: the files cv2.imwrite writes at compression 0, byte for byte): the host decodes the 8-bit input PNGs
and writes finished files, the next frame's decode on one thread and the previous frame's three writes on a small pool
while the current frame is on the GPU.

With --gpus N > 1 the script re-runs itself under `python -m torch.distributed.run --nproc-per-node N`; under torchrun
(any world size) rank t % N filters frame t and writes its concat and filter files, and rank 0 refines every frame in
order and writes the final files (run_frames_sharded).  The files are those of the one-GPU loop, byte for byte."""
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
# not in the reference: filter the frames on this many GPUs of the node, round-robin, and refine them in order on the
# first (started under torch.distributed.run; the loop under a launcher is always threaded)
parser.add_argument('--gpus', type=int, default=1)


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


def _settle(pending, keep):
    """Wait for the writes of every call in `pending` but the last `keep`."""
    while len(pending) > keep:
        for w in pending.pop(0):
            w.result()


def run_frames_sharded(stage2, content_names, style_names, out_dirs, pg, device, progress=lambda it: it, in_flight=2):
    """run_frames on one rank of the process group `pg`, writing the same files.  Rank t % world owns frame t: it
    decodes the frame on its decoder thread, runs Stage2.filter_png, writes the concat and filter files on its writer
    threads and sends P_t to rank 0 (b200.launch.send_to_root), with at most `in_flight` sends outstanding.  Rank 0
    runs the refinement chain over t = 0 ... T-1 in order, on its own P_t or the one received from the owner (shaped
    from the content file's header), and writes every final file.  Round-robin keeps the chain fed in order while a rank
    holds only a few P_t.  A rank that owns no frame returns at once."""
    import torch.distributed as dist
    from b200 import launch
    from b200.stage2 import pad_geometry
    rank, world = dist.get_rank(pg), dist.get_world_size(pg)
    n = len(content_names)
    mine = list(range(rank, n, world))
    stage2.reset()
    decoder, writers = cf.ThreadPoolExecutor(1), cf.ThreadPoolExecutor(3)
    # a half's files are views of a buffer Stage2 reuses two calls of that half later: a call's writes are awaited
    # before the call after next
    filter_writes, final_writes, sends = [], [], []
    try:
        load = lambda t: (decoder.submit(_decode, content_names[t]), decoder.submit(_decode, style_names[t]))
        nxt = load(mine[0]) if mine else None

        def filter_next(j):
            """Filter mine[j] (whose decode is in nxt) and write its two files; returns (P_t, (H, W))."""
            nonlocal nxt
            t = mine[j]
            content, style = (f.result() for f in nxt)
            nxt = load(mine[j + 1]) if j + 1 < len(mine) else None
            _settle(filter_writes, 1)
            pred, files = stage2.filter_png(content, style)
            filter_writes.append([writers.submit(_write, files[k], "{}/{:05d}.png".format(out_dirs[k], t))
                                  for k in ("concat", "filter")])
            return pred, content.shape[:2]

        if rank == 0:
            for t in progress(range(n)):
                if t % world == 0:
                    pred, size = filter_next(t // world)
                else:
                    with Image.open(content_names[t]) as im:
                        w, h = im.size
                    left, right, _, bottom = pad_geometry(h, w)
                    pred = launch.recv_on_root((1, 3, h + bottom, w + left + right), t % world, device, pg)
                    size = (h, w)
                _settle(final_writes, 1)
                final = stage2.refine_png(pred, size)
                final_writes.append([writers.submit(_write, final, "{}/{:05d}.png".format(out_dirs["final"], t))])
        else:
            for j in range(len(mine)):
                pred, _ = filter_next(j)
                if len(sends) == in_flight:
                    sends.pop(0)[0].wait()          # the oldest P_t's memory is reused only after its send
                sends.append(launch.send_to_root(pred, pg))
            for work, _ in sends:
                work.wait()
            if device.type == "cuda":
                torch.cuda.synchronize(device)
        _settle(filter_writes, 0)
        _settle(final_writes, 0)
    finally:
        decoder.shutdown(wait=True, cancel_futures=True)
        writers.shutdown(wait=True, cancel_futures=True)


def _setup(opts, device):
    """The stage of the script's networks on `device`, the content and stage-1 frame lists and the output folders."""
    seed = 2023
    np.random.seed(seed); torch.manual_seed(seed); random.seed(seed)
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
    return (Stage2(filter_net, local_net, device), content_names, style_names,
            {"concat": out_concat, "filter": out_filter, "final": out_final})


def _videos(opts, out_dirs):
    if shutil.which("ffmpeg"):
        for d in out_dirs.values():
            os.system("ffmpeg -y -r %s -i %s -crf 25 -r 12 -qscale 4  %s" % (opts.fps, os.path.join(d, "%05d.png"), d + ".mp4"))


def main(opts):
    if not torch.cuda.is_available():
        raise Exception("No GPU found, run with cpu")
    stage2, content_names, style_names, out_dirs = _setup(opts, torch.device("cuda:{}".format(opts.gpu)))
    run_frames(stage2, content_names, style_names, out_dirs, sync_io=opts.sync_io, progress=tqdm)
    _videos(opts, out_dirs)


def main_sharded(opts, device, pg):
    """main() on one rank of the process group `pg` (run_frames_sharded); after a barrier rank 0 writes the videos.
    Rank 0 prints the loop's wall time, closed by a device synchronise and a barrier, as one `stage2_loop {...}` JSON
    line."""
    import json
    import time
    import torch.distributed as dist
    rank = dist.get_rank(pg)
    stage2, content_names, style_names, out_dirs = _setup(opts, device)
    dist.barrier(pg)
    t0 = time.perf_counter()
    run_frames_sharded(stage2, content_names, style_names, out_dirs, pg, device,
                       progress=tqdm if rank == 0 else (lambda it: it))
    torch.cuda.synchronize(device)
    dist.barrier(pg)
    if rank == 0:
        print("stage2_loop " + json.dumps(dict(world=dist.get_world_size(pg), frames=len(content_names),
                                               seconds=time.perf_counter() - t0)), flush=True)
        _videos(opts, out_dirs)


if __name__ == "__main__":
    opts = parser.parse_args()
    from b200 import launch
    env = launch.torchrun_env()
    if env is None and opts.gpus > 1:
        sys.exit(launch.relaunch(__file__, sys.argv[1:], opts.gpus))
    if env is None:
        main(opts)
    else:
        device, pg = launch.init(env[2])
        main_sharded(opts, device, pg)
        launch.finish()
