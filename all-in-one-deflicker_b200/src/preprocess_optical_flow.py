"""RAFT flow pre-pass.  CLI and on-disk contract of the reference's src/preprocess_optical_flow.py: for every pair
of consecutive frames `a`, `b` in `--vid-path` it writes `<vid>_flow/a_b.npy` and `<vid>_flow/b_a.npy`, each an
(H, W, 2) float32 array, skipping pairs of which either file already exists.

The pairs are computed in windows of consecutive frames: each frame is decoded once (on a decoder thread, one window
ahead) and encoded once, a window's forward and backward flows are refined as one batch (RAFT.forward_sequence), and
the files are written on writer threads while the next window runs."""
import argparse
import concurrent.futures as cf
import os
import sys
from pathlib import Path

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
from tqdm import tqdm  # noqa: E402

DEFAULT_WEIGHTS = 'pretrained_weights/raft-things.pth'


# Window length (window_pairs): a window of K pairs holds 2K correlation states and 2K flows' refinement buffers in the
# captured graph, and K + 1 frames' encoder activations, against MEMORY_SHARE of the free device memory.
MEMORY_SHARE = 0.5
MAX_FLOWS_PER_BATCH = 16           # beyond ~3 flows at 640x360 the update-block launches already fill 132 SMs
ENCODER_BYTES_PER_PIXEL = 320      # fnet + cnet activations per frame pixel (4K pair on an H100: ~240 measured)
REFINE_BYTES_PER_PIXEL = 256       # update-block buffers of one flow in the graph pool, per frame pixel


def window_pairs(H8, W8, pairs_left, free_bytes, device_bytes, alternate_corr=False):
    """Pairs per window for feature maps of H8 x W8 with `free_bytes` of device memory free (torch.cuda.mem_get_info)
    on a device of `device_bytes`: as many as fit in MEMORY_SHARE of the free memory, at most MAX_FLOWS_PER_BATCH / 2
    and `pairs_left`, never fewer than one.  The correlation block is the one RAFT picks for that size
    (corr_block_class): batching never changes a flow's arithmetic."""
    import types
    from b200 import _native as N
    from src.models.stage_1.core.corr import AlternateCorrBlock
    from src.models.stage_1.core.raft import corr_block_class
    block = corr_block_class(types.SimpleNamespace(alternate_corr=alternate_corr), H8, W8, device_bytes)
    floats = (N.lib().b200_corr_alt_floats(256, H8, W8) if block is AlternateCorrBlock
              else N.lib().b200_corr_pyramid_floats(H8, W8))
    pixels = 64 * H8 * W8
    frame = ENCODER_BYTES_PER_PIXEL * pixels
    per_pair = frame + 2 * (4 * int(floats) + REFINE_BYTES_PER_PIXEL * pixels)
    k = int((MEMORY_SHARE * free_bytes - frame) // per_pair)
    return max(1, min(k, MAX_FLOWS_PER_BATCH // 2, pairs_left))


def window_plan(todo, k):
    """Pair indices to compute (ascending; pair p = frames p, p + 1) -> windows [first, last) of consecutive pairs
    from `todo`, each at most k long.  A window decodes frames first .. last and writes pairs first .. last - 1; a run
    of pairs is never joined across a pair that is not to be computed."""
    windows = []
    for p in todo:
        if windows and windows[-1][1] == p and p - windows[-1][0] < k:
            windows[-1][1] = p + 1
        else:
            windows.append([p, p + 1])
    return [tuple(w) for w in windows]


def flow_files(flow_dir, frames, p):
    """(forward, backward) flow file of pair p (frames p, p + 1)."""
    a, b = frames[p].name, frames[p + 1].name
    return flow_dir / '{}_{}.npy'.format(a, b), flow_dir / '{}_{}.npy'.format(b, a)


def pending_pairs(flow_dir, frames, p0, p1):
    """Pairs of [p0, p1) to compute: those of which neither flow file exists."""
    return [p for p in range(p0, p1) if not any(f.exists() for f in flow_files(flow_dir, frames, p))]


def preprocess(args, rank=0, world=1):
    """Flows of every consecutive frame pair, or of `rank`'s contiguous block of pairs when `world` ranks share the
    video.  Every thread is joined on return and on any exception."""
    import torch
    frames = sorted(args.vid_path.glob('*.*g'))                 # *.png / *.jpg / *.jpeg
    flow_dir = args.vid_path.parent / (args.vid_path.name + '_flow')
    flow_dir.mkdir(exist_ok=True)
    weights = DEFAULT_WEIGHTS
    if not os.path.exists(weights):
        # the reference dies in torch.load here (raft_wrapper.py:23); random weights would silently write garbage
        # flows that are never recomputed.  Tests that only exercise the plumbing opt in explicitly.
        if os.environ.get("B200_ALLOW_RANDOM_RAFT") != "1":
            raise FileNotFoundError(f"{weights} is missing (set B200_ALLOW_RANDOM_RAFT=1 to run with randomly "
                                    f"initialised RAFT weights, for plumbing tests only)")
        weights = None
    from src.models.stage_1.raft_wrapper import RAFTWrapper
    raft = RAFTWrapper(model_path=weights, max_long_edge=args.max_long_edge)
    p0, p1 = 0, max(len(frames) - 1, 0)
    if world > 1:
        from b200.launch import pair_block
        p0, p1 = pair_block(rank, world, len(frames))
    files = lambda p: flow_files(flow_dir, frames, p)
    todo = pending_pairs(flow_dir, frames, p0, p1)
    if not todo:
        return
    H8, W8 = raft.feature_grid(frames[todo[0]])
    free, total = torch.cuda.mem_get_info()
    k = window_pairs(H8, W8, len(todo), free, total, raft.args.alternate_corr)
    windows = window_plan(todo, k)
    decoder, writers = cf.ThreadPoolExecutor(1), cf.ThreadPoolExecutor(4)
    try:
        load = lambda w: decoder.submit(raft.load_window, [str(frames[i]) for i in range(w[0], w[1] + 1)])
        nxt, writes = load(windows[0]), []
        with tqdm(total=len(todo), desc='computing flow', disable=rank != 0) as bar:
            for j, (first, last) in enumerate(windows):
                batch = nxt.result()
                nxt = load(windows[j + 1]) if j + 1 < len(windows) else None
                fwd, bwd = raft.compute_flow_sequence(batch, pad_to=k)
                for i, p in enumerate(range(first, last)):
                    fwd_file, bwd_file = files(p)
                    writes += [writers.submit(np.save, fwd_file, fwd[i]), writers.submit(np.save, bwd_file, bwd[i])]
                bar.update(last - first)
        for w in writes:
            w.result()
    finally:
        decoder.shutdown(wait=True, cancel_futures=True)
        writers.shutdown(wait=True, cancel_futures=True)


def preprocess_sharded(vid_path, rank, world, max_long_edge=2000):
    """`rank`'s block of the pre-pass, then a barrier of the process group: every flow file exists on return."""
    import torch
    import torch.distributed as dist
    preprocess(argparse.Namespace(vid_path=Path(vid_path), max_long_edge=max_long_edge), rank, world)
    torch.cuda.empty_cache()
    dist.barrier()


if __name__ == '__main__':
    cli = argparse.ArgumentParser(description='Preprocess image sequence')
    cli.add_argument('--vid-path', type=Path, default=Path('./data/'), help='folder to process')
    cli.add_argument('--max_long_edge', type=int, default=2000)
    cli.add_argument('--gpu', type=int, default=0)
    cli.add_argument('--gpus', type=int, default=1, help='split the frame pairs over this many GPUs of the node')
    opts = cli.parse_args()
    from b200 import launch
    env = launch.torchrun_env()
    if env is None and opts.gpus > 1:
        sys.exit(launch.relaunch(__file__, sys.argv[1:], opts.gpus))
    if env is None:
        os.environ["CUDA_VISIBLE_DEVICES"] = str(opts.gpu)
        preprocess(opts)
    else:
        launch.init(env[2])
        preprocess_sharded(opts.vid_path, env[0], env[1], opts.max_long_edge)
        launch.finish()
