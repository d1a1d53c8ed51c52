"""Stage 1, segmentation variant — fit a two-layer neural atlas (foreground / background + alpha) of one video.  Same
CLI, config keys, on-disk inputs and outputs as the reference script (src/stage1_neural_atlas_seg.py:320-368); the
loop body (:195-319) runs in libb200deflicker.so (b200_seg_loss_grad + b200_adam_step).

    python src/stage1_neural_atlas_seg.py --vid_name NAME --class_name portrait [--config config_flow_100.json]
                                          [--root data/test/] [--down 1] [--gpu 0] [--gpus 1]
                                          [--clips [--clip_overlap V]]

With --gpus N > 1 the script re-runs itself under `python -m torch.distributed.run --nproc-per-node N`; under torchrun
(any world size) every rank computes a block of the flow pairs, holds a block of the frames and their mattes and
evaluates those frames.

With --clips a video longer than maximum_number_of_frames is fitted as clips (b200.atlas.clip_plan), one atlas each,
the clips spread over the ranks under torchrun; see `fit_clips`.  With --clip_overlap V consecutive clips share V
frames, which are written once every clip is fitted as a cross-fade of the two atlases' renders; see `stitch`.

The mattes of `<root>/<NAME>_seg/` are an input: the reference produces them with third-party models (CarveKit /
detectron2 Mask-RCNN, src/preprocess_mask_*.py) that this repository does not ship; the script stops with a clear
message when they are missing.
"""
import argparse
import gc
import glob
import json
import os
import subprocess
import sys
from pathlib import Path

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

import cv2          # noqa: E402
import numpy as np  # noqa: E402
import torch        # noqa: E402
from tqdm import tqdm  # noqa: E402

from b200 import _native as N  # noqa: E402
from b200 import atlas as A    # noqa: E402
from b200 import seg as SG     # noqa: E402
from src.models.stage_1.evaluate import evaluate_model, stitch_seams  # noqa: E402
from src.models.stage_1.unwrap_utils import load_mask_frames, mask_files, pre_train_mapping  # noqa: E402


def frame_size(args):
    """(resx, resy) the video is fitted at: its first frame's size divided by --down."""
    frames_list = sorted(glob.glob(os.path.join(args.vid_path, "*g")))
    first = cv2.imread(frames_list[0])
    resx, resy = first.shape[1], first.shape[0]
    if args.down is not None:
        resx, resy = int(resx / args.down), int(resy / args.down)
    return resx, resy


def main(config, args, clip=None, device=None, own=None):
    """Fit the two-layer atlas of the video on `device` (default: the current CUDA device).  With `clip` = (c0, c1):
    the run on a folder holding only frames [c0, c1), their flows and their mattes, its files under
    stage_1/clip_<c0>_<c1>/ except the output frames, which go to stage_1/output/ at their frame numbers in the whole
    video; with `own` = (a, b) the output frames of [a, b) only (the frames the clip shares with no other clip)."""
    resx, resy = frame_size(args)
    data_folder = Path(args.vid_path)
    vid_name, vid_root = data_folder.name, data_folder.parent
    stage_folder = Path(f'./results/{vid_name}/stage_1')
    results_folder = stage_folder if clip is None else stage_folder / A.clip_name(clip)
    output = {} if clip is None else dict(output_folder=str(stage_folder / "output"), frame_offset=clip[0])
    if own is not None:
        output["write_frames"] = range(own[0] - clip[0], own[1] - clip[0])
    results_folder.mkdir(parents=True, exist_ok=True)
    with open('%s/config.json' % results_folder, 'w') as f:
        json.dump(config, f, indent=4)

    device = torch.device("cuda") if device is None else device
    video, frames = A.DeviceVideo.from_files(data_folder, vid_root, vid_name, resy, resx,
                                             config["maximum_number_of_frames"], device, filter_optical_flow=True,
                                             clip=clip)
    T = frames.shape[3]
    mask_frames = load_mask_frames(resy, resx, T, vid_root, vid_name, clip=clip)
    precision = N.PREC_TC if N.lib().b200_device_supports_tc() else N.PREC_FP32
    trainer = SG.SegTrainer(video, SG.pack_mask_frames(mask_frames, device), config, precision=precision, device=device,
                            resx=resx)
    trainer.init_like_reference()          # mapping1, mapping2, atlas, alpha: nn.Linear stream order (:127-161)

    start_iteration = 0
    larger_dim = np.maximum(resx, resy)
    if not config["load_checkpoint"]:
        for which in ("mapping1", "mapping2"):
            if config["pretrain_" + which]:
                pre_train_mapping(trainer, T, config["uv_mapping_scale"], resx=resx, resy=resy, larger_dim=larger_dim,
                                  device=device, pretrain_iters=config["pretrain_iter_number"], which=which)
    else:
        ck = torch.load(config["checkpoint_path"])
        trainer.load_state(dict(atlas=ck["F_atlas_state_dict"], mapping1=ck["model_F_mapping1_state_dict"],
                                mapping2=ck["model_F_mapping2_state_dict"], alpha=ck["model_F_alpha_state_dict"]))
        trainer.load_optimizer_state_dict(ck["optimizer_all_state_dict"])
        start_iteration = ck["iteration"]

    n_pixels = T * resy * resx
    samples = int(config["samples_batch"])
    evaluate_every = int(config["evaluate_every"])
    for i in tqdm(range(start_iteration, config["iters_num"])):
        inds = torch.randint(n_pixels, (samples, 1))       # same CPU-generator draw as the reference (:204)
        trainer.step_host(inds, i)
        if i % evaluate_every == 0 and i > start_iteration:
            evaluate_model(trainer, resx, resy, T, frames, results_folder, i, mask_frames, vid_name, **output)
    trainer.release()


def fit_clips(config, args, clips, device, seed, overlap=0):
    """Fit one two-layer atlas per clip of `clips` on `device`, in order, with no process group: clip k is
    `main(config, args, clip)`, started from the CPU generator seeded with `seed`, so its files are those of a
    stand-alone run on a folder holding only its frames and mattes.  Nothing of a clip is alive when the next one is
    loaded.  With `overlap` V > 0 (clips of clip_plan(T, M, V)) a clip leaves the output frames it shares with a
    neighbour to `stitch`."""
    n_frames = len(A.video_files(args.vid_path))
    for clip in clips:
        torch.manual_seed(seed)
        with torch.cuda.device(device):
            main(config, args, clip, device, A.clip_own_frames(clip, n_frames, overlap) if overlap > 0 else None)
            gc.collect()
            torch.cuda.empty_cache()


def stitch(config, args, plan, device, rank=0, world=1):
    """The frames consecutive clips of `plan` share (--clip_overlap), for the seams rank `rank` of `world` owns:
    stitch_seams with render-only SegTrainers loaded from the clips' checkpoints, in the precision of the clips'
    evaluations."""
    resx, resy = frame_size(args)
    precision = N.PREC_TC if N.lib().b200_device_supports_tc() else N.PREC_FP32

    def make_trainer(path):
        ck = torch.load(path, map_location="cpu")
        trainer = SG.SegTrainer(None, None, config, precision=precision, device=device, resx=resx)
        trainer.load_state(dict(atlas=ck["F_atlas_state_dict"], mapping1=ck["model_F_mapping1_state_dict"],
                                mapping2=ck["model_F_mapping2_state_dict"], alpha=ck["model_F_alpha_state_dict"]))
        return trainer
    with torch.cuda.device(device):
        return stitch_seams(plan, make_trainer, Path(f'./results/{Path(args.vid_path).name}/stage_1'), resx, resy,
                            rank, world)


def check_clip_mattes(vid_path, clips):
    """Refuse, naming the first clip concerned, a matte folder that holds fewer mattes than the video has frames."""
    data_folder = Path(vid_path)
    for clip in clips:
        mask_files(data_folder.parent, data_folder.name, clip[1] - clip[0], clip)


def main_sharded(config, args, device, pg):
    """`main` on one rank of a process group: this rank's frame block and matte resident, the exchange of SegTrainer,
    the evaluation sharded by frame.  Every rank draws rank 0's random stream and pre-trains in full."""
    import torch.distributed as dist
    from b200 import launch
    from src.models.stage_1.evaluate import evaluate_model_sharded
    rank, world = dist.get_rank(pg), dist.get_world_size(pg)
    resx, resy = frame_size(args)
    data_folder = Path(args.vid_path)
    vid_name, vid_root = data_folder.name, data_folder.parent
    results_folder = Path(f'./results/{vid_name}/stage_1')
    results_folder.mkdir(parents=True, exist_ok=True)
    if rank == 0:
        with open('%s/config.json' % results_folder, 'w') as f:
            json.dump(config, f, indent=4)
    T = int(min(config["maximum_number_of_frames"], len(A.video_files(data_folder))))
    t_begin, t_end = A.frame_range(rank, world, T)
    video, _ = A.DeviceVideo.from_files(data_folder, vid_root, vid_name, resy, resx, config["maximum_number_of_frames"],
                                        device, filter_optical_flow=True, t_begin=t_begin, t_end=t_end, decode_all=False)
    mask_frames = load_mask_frames(resy, resx, T, vid_root, vid_name)
    precision = N.PREC_TC if N.lib().b200_device_supports_tc() else N.PREC_FP32
    trainer = SG.SegTrainer(video, SG.pack_mask_frames(mask_frames, device, t_begin, t_end), config, precision=precision,
                            device=device, resx=resx, process_group=pg)
    launch.shared_seed(pg)
    trainer.init_like_reference()

    start_iteration = 0
    larger_dim = np.maximum(resx, resy)
    if not config["load_checkpoint"]:
        for which in ("mapping1", "mapping2"):
            if config["pretrain_" + which]:
                pre_train_mapping(trainer, T, config["uv_mapping_scale"], resx=resx, resy=resy, larger_dim=larger_dim,
                                  device=device, pretrain_iters=config["pretrain_iter_number"], which=which)
    else:
        ck = torch.load(config["checkpoint_path"], map_location="cpu")
        trainer.load_state(dict(atlas=ck["F_atlas_state_dict"], mapping1=ck["model_F_mapping1_state_dict"],
                                mapping2=ck["model_F_mapping2_state_dict"], alpha=ck["model_F_alpha_state_dict"]))
        trainer.load_optimizer_state_dict(ck["optimizer_all_state_dict"])
        start_iteration = ck["iteration"]
    launch.broadcast_params(trainer.params, pg)

    n_pixels = T * resy * resx
    samples = int(config["samples_batch"])
    evaluate_every = int(config["evaluate_every"])
    for i in tqdm(range(start_iteration, config["iters_num"]), disable=rank != 0):
        inds = torch.randint(n_pixels, (samples, 1))
        if i == start_iteration:
            launch.check_replicas(pg, parameters=trainer.params, first_index_batch=inds)
        trainer.step_host(inds, i)
        if i % evaluate_every == 0 and i > start_iteration:
            evaluate_model_sharded(trainer, resx, resy, T, results_folder, i, vid_name, process_group=pg)


if __name__ == "__main__":
    parser = argparse.ArgumentParser()
    parser.add_argument('--config', type=str, default="config_flow_100.json")
    parser.add_argument('--vid_name', type=str, default="Around_the_world_in_1896_001")
    parser.add_argument('--root', type=str, default="data/test/")
    parser.add_argument('--down', type=int, default=1)
    parser.add_argument('--gpu', type=str, default="0")
    parser.add_argument('--class_name', type=str, default="portrait")
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
    from b200 import launch
    env = launch.torchrun_env()
    if env is None and args.gpus > 1:
        sys.exit(launch.relaunch(__file__, sys.argv[1:], args.gpus))
    args.vid_path = os.path.join(args.root, args.vid_name)
    seg_dir = args.vid_path.rstrip("/") + "_seg"
    with open(os.path.join(HERE, "config", args.config)) as f:
        config = json.load(f)
    clips = A.video_clips(config, len(A.video_files(args.vid_path)), args.clip_overlap) if args.clips else [None]
    if env is not None:
        if not glob.glob(os.path.join(seg_dir, "*g")):
            raise FileNotFoundError(f"{seg_dir} holds no mattes: produce them with the reference's mask pre-pass "
                                    f"(class '{args.class_name}') or any segmentation tool, one image per frame")
        from src.preprocess_optical_flow import preprocess_sharded
        device, pg = launch.init(env[2])
        preprocess_sharded(args.vid_path, env[0], env[1])
        if len(clips) > 1:
            check_clip_mattes(args.vid_path, clips)
            seed, done = launch.shared_seed(pg), launch.patient_group()
            fit_clips(config, args, A.rank_clips(clips, env[0], env[1]), device, seed, args.clip_overlap)
            torch.distributed.barrier(group=done)
            if args.clip_overlap > 0:
                stitch(config, args, clips, device, env[0], env[1])
                torch.distributed.barrier(group=done)
        else:
            main_sharded(config, args, device, pg)
        launch.finish()
        sys.exit(0)
    os.environ["CUDA_VISIBLE_DEVICES"] = args.gpu
    cmd = "%s %s --vid-path %s --gpu %s " % (sys.executable, os.path.join(HERE, "preprocess_optical_flow.py"),
                                             args.vid_path, args.gpu)
    print(cmd)
    if subprocess.call(cmd, shell=True) != 0:
        raise RuntimeError("optical-flow pre-pass failed")
    if not glob.glob(os.path.join(seg_dir, "*g")):
        raise FileNotFoundError(f"{seg_dir} holds no mattes: produce them with the reference's mask pre-pass "
                                f"(class '{args.class_name}') or any segmentation tool, one image per frame")
    if len(clips) > 1:
        check_clip_mattes(args.vid_path, clips)
        fit_clips(config, args, clips, torch.device("cuda"), torch.initial_seed(), args.clip_overlap)
        if args.clip_overlap > 0:
            stitch(config, args, clips, torch.device("cuda"))
    else:
        main(config, args)
