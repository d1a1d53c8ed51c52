"""The run of both stage-1 scripts (src/stage1_neural_atlas.py, src/stage1_neural_atlas_seg.py): the command line, the
flow pre-pass, the whole-video, frame-sharded and clip fits, the stitch of overlapping clips.  A script passes its
`Variant`, which holds everything the two variants do differently; nothing here depends on which variant it is."""
import argparse
import gc
import glob
import json
import os
import subprocess
import sys
from pathlib import Path

import cv2
import torch
import torch.distributed as dist
from tqdm import tqdm

from b200 import _native as N
from b200 import atlas as A
from b200 import launch
from src.models.stage_1.evaluate import stitch_seams
from src.models.stage_1.unwrap_utils import pre_train_mapping, save_mask_flow

SRC = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


class Variant:
    """What a stage-1 variant adds to the run.  A script subclasses it and implements:

    `trainer(video, config, vid_path=None, clip=None, **kw)`: the variant's FlatTrainer of the DeviceVideo `video` of
    the folder `vid_path` (frames [c0, c1) of it with `clip`), or a render-only trainer when `video` is None; `kw` are
    the trainer's precision, device, resx and process_group.
    `evaluate(trainer, resx, resy, T, frames, folder, it, vid_name, artefacts, writer, **output)`: the whole-video or
    clip evaluation of iteration `it` against the decoded `frames`, `output` its output_folder, frame_offset and
    write_frames.
    `evaluate_sharded(trainer, resx, resy, T, folder, it, vid_name, artefacts, writer, pg)`: the same, collective over
    the ranks of `pg`, each evaluating its own frames.
    """

    pretrain = {}       # the networks pre-trained before the loop, in order: {pre_train_mapping's `which`: config flag}

    def artefacts(self, args):
        """Whether the run writes the evaluation videos, the tensorboard log and the mask-flow videos."""
        return False

    def check_inputs(self, args):
        """Refuse a video the variant cannot fit (after the flow pre-pass; under torchrun before the ranks meet)."""

    def check_clips(self, vid_path, clips):
        """Refuse a `--clips` run the variant cannot fit, before any clip is fitted."""


def frame_size(vid_path, down):
    """(resx, resy) the video is fitted at: its first frame's size divided by `down`."""
    first = cv2.imread(sorted(glob.glob(os.path.join(vid_path, "*g")))[0])
    resx, resy = first.shape[1], first.shape[0]
    if down is not None:
        resx, resy = int(resx / down), int(resy / down)
    return resx, resy


def precision():
    """The precision of every stage-1 trainer: the tensor cores where the device has them."""
    return N.PREC_TC if N.lib().b200_device_supports_tc() else N.PREC_FP32


def fit(variant, config, args, device, pg=None, clip=None, own=None, phases=None):
    """Fit the variant's atlas of the video `args.vid_path` on `device`.

    With no process group: the whole video, or with `clip` = (c0, c1) the run on a folder holding only frames [c0, c1)
    (and their flows and mattes), its files under stage_1/clip_<c0>_<c1>/ except the output frames, which go to
    stage_1/output/ at their frame numbers in the whole video; with `own` = (a, b) the output frames of [a, b) only
    (the frames the clip shares with no other clip).

    With a process group `pg`: one rank of the frame-sharded fit.  The rank holds its own block of frames, the trainer
    exchanges gradients between the ranks, every rank draws rank 0's random stream and pre-trains in full, and the
    evaluation is sharded by frame.  `phases` (launch.Phases) accumulates the wall time of loading, pre-training, the
    loop and the evaluation, and reports it."""
    rank, world = (0, 1) if pg is None else (dist.get_rank(pg), dist.get_world_size(pg))
    mark = phases.mark if phases is not None else lambda name: None
    resx, resy = frame_size(args.vid_path, args.down)
    data_folder = Path(args.vid_path)
    vid_name, vid_root = data_folder.name, data_folder.parent
    stage_folder = Path(f'./results/{vid_name}/stage_1')
    results_folder = stage_folder if clip is None else stage_folder / A.clip_name(clip)
    output = {} if clip is None else dict(output_folder=str(stage_folder / "output"), frame_offset=clip[0])
    if own is not None:
        output["write_frames"] = range(own[0] - clip[0], own[1] - clip[0])
    results_folder.mkdir(parents=True, exist_ok=True)
    if rank == 0:
        with open('%s/config.json' % results_folder, 'w') as f:
            json.dump(config, f, indent=4)

    if clip is None:
        T = int(min(config["maximum_number_of_frames"], len(A.video_files(data_folder))))
    else:
        T = clip[1] - clip[0]
    t_begin, t_end = A.frame_range(rank, world, T)
    artefacts = variant.artefacts(args)
    # input producer on the device (the reference's load_input_data_single, unwrap_utils.py:105-163): frames, image
    # differences, resized flows and consistency masks go straight into HBM.  `frames`, the decoded video, is for the
    # host PSNR of the whole-video evaluation; a frame shard decodes its own frames only, and rank 0 decodes them all
    # for the startup videos
    video, frames = A.DeviceVideo.from_files(data_folder, vid_root, vid_name, resy, resx,
                                             config["maximum_number_of_frames"], device, filter_optical_flow=True,
                                             t_begin=t_begin, t_end=t_end,
                                             decode_all=pg is None or (rank == 0 and artefacts), clip=clip)
    mark("load")
    writer = None
    if rank == 0 and artefacts:    # the reference's tensorboard log + overview videos (:99,109; unwrap_utils.py:200-231)
        from torch.utils.tensorboard import SummaryWriter
        writer = SummaryWriter(log_dir=str(results_folder))
        save_mask_flow(video.mask_fwd_host(), frames, results_folder)
    if pg is not None:
        frames = None
    trainer = variant.trainer(video, config, vid_path=args.vid_path, clip=clip, precision=precision(), device=device,
                              resx=resx, process_group=pg)
    if pg is not None:
        launch.shared_seed(pg)
    trainer.init_like_reference()          # nn.Linear's stream order in CONSTRUCTION_ORDER

    start_iteration = 0
    if config["load_checkpoint"]:
        start_iteration = trainer.load_checkpoint(torch.load(config["checkpoint_path"], map_location="cpu"))
    else:
        for which, flag in variant.pretrain.items():
            if config[flag]:
                pre_train_mapping(trainer, T, config["uv_mapping_scale"], resx=resx, resy=resy,
                                  larger_dim=max(resx, resy), device=device,
                                  pretrain_iters=config["pretrain_iter_number"], which=which)
    if pg is not None:
        launch.broadcast_params(trainer.params, pg)
    mark("pretrain")

    n_pixels = T * resy * resx
    samples = int(config["samples_batch"])
    evaluate_every = int(config["evaluate_every"])
    for i in tqdm(range(start_iteration, config["iters_num"]), disable=rank != 0):
        inds = torch.randint(n_pixels, (samples, 1))       # same CPU-generator draw as the reference (:159)
        if pg is not None and i == start_iteration:
            launch.check_replicas(pg, parameters=trainer.params, first_index_batch=inds)
        trainer.step_host(inds, i)
        if i % evaluate_every == 0 and i > start_iteration:
            mark("loop")
            if pg is None:
                variant.evaluate(trainer, resx, resy, T, frames, results_folder, i, vid_name, artefacts, writer,
                                 **output)
            else:
                variant.evaluate_sharded(trainer, resx, resy, T, results_folder, i, vid_name, artefacts, writer, pg)
            mark("evaluation")
    mark("loop")
    if phases is not None:
        phases.report()
    if writer is not None:
        writer.close()
    if pg is None:
        trainer.release()


def fit_clips(variant, config, args, clips, device, seed, overlap=0):
    """Fit one atlas per clip of `clips` on `device`, in order, with no process group: clip k is `fit` of that clip,
    started from the CPU generator seeded with `seed`, so its files are those of a stand-alone run on a folder holding
    only its frames (and mattes).  Nothing of a clip is alive when the next one is loaded.  With `overlap` V > 0 (clips
    of clip_plan(T, M, V)) a clip leaves the output frames it shares with a neighbour to `stitch`."""
    n_frames = len(A.video_files(args.vid_path))
    for clip in clips:
        torch.manual_seed(seed)
        with torch.cuda.device(device):
            fit(variant, config, args, device, clip=clip,
                own=A.clip_own_frames(clip, n_frames, overlap) if overlap > 0 else None)
            gc.collect()
            torch.cuda.empty_cache()


def stitch(variant, config, args, plan, device, rank=0, world=1):
    """The frames consecutive clips of `plan` share (--clip_overlap), for the seams rank `rank` of `world` owns:
    stitch_seams with the variant's render-only trainers loaded from the clips' checkpoints, in the precision of the
    clips' evaluations."""
    resx, resy = frame_size(args.vid_path, args.down)

    def make_trainer(path):
        trainer = variant.trainer(None, config, precision=precision(), device=device, resx=resx)
        trainer.load_checkpoint(torch.load(path, map_location="cpu"), optimizer=False)
        return trainer
    with torch.cuda.device(device):
        return stitch_seams(plan, make_trainer, Path(f'./results/{Path(args.vid_path).name}/stage_1'), resx, resy,
                            rank, world)


def parse_args(add_flags):
    """The command line of a stage-1 script: the flags both take, with `add_flags(parser)` adding the script's own
    after --root."""
    parser = argparse.ArgumentParser()
    parser.add_argument('--config', type=str, default="config_flow_100.json")
    parser.add_argument('--vid_name', type=str, default="Around_the_world_in_1896_001")
    parser.add_argument('--root', type=str, default="data/test/")
    add_flags(parser)
    parser.add_argument('--gpus', type=int, default=1,
                        help="fit on this many GPUs of the node, the video sharded by frame (started under torchrun)")
    parser.add_argument('--clips', action='store_true',
                        help="fit a video longer than maximum_number_of_frames as clips of at most that many frames, "
                             "one atlas each (spread over the GPUs with --gpus)")
    parser.add_argument('--clip_overlap', type=int, default=0,
                        help="with --clips: consecutive clips share this many frames, written as a cross-fade of the "
                             "two atlases' renders")
    args = parser.parse_args()
    if args.clip_overlap != 0 and not args.clips:
        parser.error("--clip_overlap is only meaningful with --clips")
    return args


def run(variant, args):
    """A stage-1 script on the command line `args`.  With --gpus N > 1 and no launcher the script re-runs itself under
    torch.distributed.run.  Under torchrun (any world size) every rank computes a block of the flow pairs, then fits
    its frame block of the video, or with --clips its clips (k = rank mod N) and its seams.  Otherwise the process runs
    the flow pre-pass on --gpu and fits the video, or its clips one after the other and then the seams."""
    env = launch.torchrun_env()
    if env is None and args.gpus > 1:
        sys.exit(launch.relaunch(sys.argv[0], sys.argv[1:], args.gpus))
    args.vid_path = os.path.join(args.root, args.vid_name)
    with open(os.path.join(SRC, "config", args.config)) as f:
        config = json.load(f)
    clips = A.video_clips(config, len(A.video_files(args.vid_path)), args.clip_overlap) if args.clips else [None]
    if env is not None:
        rank, world, local_rank = env
        variant.check_inputs(args)
        from src.preprocess_optical_flow import preprocess_sharded
        device, pg = launch.init(local_rank)
        phases = launch.Phases(pg)
        preprocess_sharded(args.vid_path, rank, world)
        if len(clips) > 1:
            variant.check_clips(args.vid_path, clips)
            seed, done = launch.shared_seed(pg), launch.patient_group()
            fit_clips(variant, config, args, A.rank_clips(clips, rank, world), device, seed, args.clip_overlap)
            dist.barrier(group=done)
            if args.clip_overlap > 0:
                stitch(variant, config, args, clips, device, rank, world)
                dist.barrier(group=done)
        else:
            phases.mark("prepass")
            fit(variant, config, args, device, pg, phases=phases)
        launch.finish()
        sys.exit(0)
    os.environ["CUDA_VISIBLE_DEVICES"] = str(args.gpu)
    # always run the pre-pass (reference :276-278): it skips the pairs whose files already exist, so a partially
    # written flow folder is completed instead of crashing later in load_input_data_single
    cmd = "%s %s --vid-path %s --gpu %s " % (sys.executable, os.path.join(SRC, "preprocess_optical_flow.py"),
                                             args.vid_path, args.gpu)
    print(cmd)
    if subprocess.call(cmd, shell=True) != 0:
        raise RuntimeError("optical-flow pre-pass failed")
    variant.check_inputs(args)
    device = torch.device("cuda")
    if len(clips) > 1:
        variant.check_clips(args.vid_path, clips)
        fit_clips(variant, config, args, clips, device, torch.initial_seed(), args.clip_overlap)
        if args.clip_overlap > 0:
            stitch(variant, config, args, clips, device)
    else:
        fit(variant, config, args, device)
