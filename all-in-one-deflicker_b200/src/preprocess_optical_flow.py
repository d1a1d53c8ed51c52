"""RAFT flow pre-pass.  CLI and on-disk contract of the reference's src/preprocess_optical_flow.py: for every pair
of consecutive frames `a`, `b` in `--vid-path` it writes `<vid>_flow/a_b.npy` and `<vid>_flow/b_a.npy`, each an
(H, W, 2) float32 array, skipping pairs that already exist.  Both directions share one feature-encoder pass."""
import argparse
import os
import sys
from pathlib import Path

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
from tqdm import tqdm  # noqa: E402

DEFAULT_WEIGHTS = 'pretrained_weights/raft-things.pth'


def preprocess(args, rank=0, world=1):
    """Flows of every consecutive frame pair, or of `rank`'s contiguous block of pairs when `world` ranks share the
    video."""
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
    pairs = list(zip(frames, frames[1:]))
    if world > 1:
        from b200.launch import pair_block
        p0, p1 = pair_block(rank, world, len(frames))
        pairs = pairs[p0:p1]
    for prev, nxt in tqdm(pairs, desc='computing flow', disable=rank != 0):
        fwd_file = flow_dir / '{}_{}.npy'.format(prev.name, nxt.name)
        bwd_file = flow_dir / '{}_{}.npy'.format(nxt.name, prev.name)
        if fwd_file.exists() or bwd_file.exists():
            continue
        im_a, im_b = raft.load_images(str(prev), str(nxt))
        fwd, bwd = raft.compute_flow_both(im_a, im_b)
        np.save(fwd_file, fwd)
        np.save(bwd_file, bwd)


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
