"""Stage 1 — fit the neural atlas of one video.  Same CLI, config keys, on-disk inputs and outputs as
the reference script (src/stage1_neural_atlas.py:257-281); the optimisation loop itself
(:151-231) runs as one replayed CUDA graph per iteration in libb200deflicker.so.

    python src/stage1_neural_atlas.py --vid_name NAME [--config config_flow_100.json] [--root data/test/]
                                      [--down 4] [--gpu 0] [--gpus 1]

With --gpus N > 1 the script re-runs itself under `python -m torch.distributed.run --nproc-per-node N`; under torchrun
(any world size) every rank computes a block of the flow pairs, holds a block of the frames and evaluates those.
"""
import argparse
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
from src.models.stage_1.evaluate import evaluate_model_single  # noqa: E402
from src.models.stage_1.unwrap_utils import pre_train_mapping, save_mask_flow  # noqa: E402


def main(config, args):
    frames_list = sorted(glob.glob(os.path.join(args.vid_path, "*g")))
    first = cv2.imread(frames_list[0])
    resx, resy = first.shape[1], first.shape[0]
    if args.down is not None:
        resx, resy = int(resx / args.down), int(resy / args.down)
    data_folder = Path(args.vid_path)
    vid_name, vid_root = data_folder.name, data_folder.parent
    results_folder = Path(f'./results/{vid_name}/stage_1')
    results_folder.mkdir(parents=True, exist_ok=True)
    with open('%s/config.json' % results_folder, 'w') as f:
        json.dump(config, f, indent=4)

    device = torch.device("cuda")
    # input producer on the device (the reference's load_input_data_single, unwrap_utils.py:105-163): frames, image
    # differences, resized flows and consistency masks go straight into HBM; `frames` is the decoded video for PSNR
    video, frames = A.DeviceVideo.from_files(data_folder, vid_root, vid_name, resy, resx,
                                             config["maximum_number_of_frames"], device, filter_optical_flow=True)
    T = frames.shape[3]
    writer = None
    if not args.no_artefacts:      # the reference's tensorboard log + overview videos (:99,109; unwrap_utils.py:200-231)
        from torch.utils.tensorboard import SummaryWriter
        writer = SummaryWriter(log_dir=str(results_folder))
        save_mask_flow(video.mask_fwd_host(), frames, results_folder)
    precision = N.PREC_TC if N.lib().b200_device_supports_tc() else N.PREC_FP32
    trainer = A.AtlasTrainer(video, config, precision=precision, device=device, resx=resx)
    trainer.init_like_reference()          # mapping then atlas, nn.Linear stream order (:112-128)

    start_iteration = 0
    larger_dim = np.maximum(resx, resy)
    if not config["load_checkpoint"]:
        if config["pretrain_mapping1"]:
            pre_train_mapping(trainer, T, config["uv_mapping_scale"], resx=resx, resy=resy, larger_dim=larger_dim,
                              device=device, pretrain_iters=config["pretrain_iter_number"])
    else:
        ck = torch.load(config["checkpoint_path"])
        trainer.load_state(ck["model_F_mapping1_state_dict"], ck["F_atlas_state_dict"])
        trainer.load_optimizer_state_dict(ck["optimizer_all_state_dict"])
        start_iteration = ck["iteration"]

    n_pixels = T * resy * resx
    samples = int(config["samples_batch"])
    evaluate_every = int(config["evaluate_every"])
    for i in tqdm(range(start_iteration, config["iters_num"])):
        inds = torch.randint(n_pixels, (samples, 1))       # same CPU-generator draw as the reference (:159)
        trainer.step_host(inds, i)
        if i % evaluate_every == 0 and i > start_iteration:
            evaluate_model_single(trainer, resx, resy, T, frames, results_folder, i, vid_name,
                                  artefacts=not args.no_artefacts, writer=writer)


def main_sharded(config, args, device, pg, phases=None):
    """`main` on one rank of a process group: this rank's frame block resident, the exchange of AtlasTrainer, the
    evaluation sharded by frame.  Every rank draws rank 0's random stream and pre-trains in full.  `phases`
    (launch.Phases) accumulates the wall time of loading, pre-training, the loop and the evaluation."""
    import torch.distributed as dist
    from b200 import launch
    from src.models.stage_1.evaluate import evaluate_model_single_sharded
    rank, world = dist.get_rank(pg), dist.get_world_size(pg)
    phases = phases or launch.Phases(pg)
    frames_list = sorted(glob.glob(os.path.join(args.vid_path, "*g")))
    first = cv2.imread(frames_list[0])
    resx, resy = first.shape[1], first.shape[0]
    if args.down is not None:
        resx, resy = int(resx / args.down), int(resy / args.down)
    data_folder = Path(args.vid_path)
    vid_name, vid_root = data_folder.name, data_folder.parent
    results_folder = Path(f'./results/{vid_name}/stage_1')
    results_folder.mkdir(parents=True, exist_ok=True)
    if rank == 0:
        with open('%s/config.json' % results_folder, 'w') as f:
            json.dump(config, f, indent=4)
    T = int(min(config["maximum_number_of_frames"], len(A.video_files(data_folder))))
    t_begin, t_end = A.frame_range(rank, world, T)
    artefacts = not args.no_artefacts
    # a rank decodes its own frames only; rank 0 also decodes the others for the startup videos
    video, frames = A.DeviceVideo.from_files(data_folder, vid_root, vid_name, resy, resx, config["maximum_number_of_frames"],
                                             device, filter_optical_flow=True, t_begin=t_begin, t_end=t_end,
                                             decode_all=rank == 0 and artefacts)
    phases.mark("load")
    writer = None
    if rank == 0 and artefacts:
        from torch.utils.tensorboard import SummaryWriter
        writer = SummaryWriter(log_dir=str(results_folder))
        save_mask_flow(video.mask_fwd_host(), frames, results_folder)
        del frames
    precision = N.PREC_TC if N.lib().b200_device_supports_tc() else N.PREC_FP32
    trainer = A.AtlasTrainer(video, config, precision=precision, device=device, resx=resx, process_group=pg)
    launch.shared_seed(pg)
    trainer.init_like_reference()

    start_iteration = 0
    larger_dim = np.maximum(resx, resy)
    if not config["load_checkpoint"]:
        if config["pretrain_mapping1"]:
            pre_train_mapping(trainer, T, config["uv_mapping_scale"], resx=resx, resy=resy, larger_dim=larger_dim,
                              device=device, pretrain_iters=config["pretrain_iter_number"])
    else:
        ck = torch.load(config["checkpoint_path"], map_location="cpu")
        trainer.load_state(ck["model_F_mapping1_state_dict"], ck["F_atlas_state_dict"])
        trainer.load_optimizer_state_dict(ck["optimizer_all_state_dict"])
        start_iteration = ck["iteration"]
    launch.broadcast_params(trainer.params, pg)
    phases.mark("pretrain")

    n_pixels = T * resy * resx
    samples = int(config["samples_batch"])
    evaluate_every = int(config["evaluate_every"])
    for i in tqdm(range(start_iteration, config["iters_num"]), disable=rank != 0):
        inds = torch.randint(n_pixels, (samples, 1))
        if i == start_iteration:
            launch.check_replicas(pg, parameters=trainer.params, first_index_batch=inds)
        trainer.step_host(inds, i)
        if i % evaluate_every == 0 and i > start_iteration:
            phases.mark("loop")
            evaluate_model_single_sharded(trainer, resx, resy, T, results_folder, i, vid_name, artefacts=artefacts,
                                          writer=writer, process_group=pg)
            phases.mark("evaluation")
    phases.mark("loop")
    phases.report()
    if writer is not None:
        writer.close()


if __name__ == "__main__":
    parser = argparse.ArgumentParser()
    parser.add_argument('--config', type=str, default="config_flow_100.json")
    parser.add_argument('--vid_name', type=str, default="Around_the_world_in_1896_001")
    parser.add_argument('--root', type=str, default="data/test/")
    parser.add_argument('--down', type=int, default=4)
    parser.add_argument('--gpu', type=int, default=0)
    parser.add_argument('--no_artefacts', action='store_true',
                        help="skip the evaluation videos / tensorboard log (checkpoint, output frames and PSNR only)")
    parser.add_argument('--gpus', type=int, default=1,
                        help="fit on this many GPUs of the node, the video sharded by frame (started under torchrun)")
    args = parser.parse_args()
    from b200 import launch
    env = launch.torchrun_env()
    if env is None and args.gpus > 1:
        sys.exit(launch.relaunch(__file__, sys.argv[1:], args.gpus))
    args.vid_path = os.path.join(args.root, args.vid_name)
    if env is not None:
        from src.preprocess_optical_flow import preprocess_sharded
        device, pg = launch.init(env[2])
        phases = launch.Phases(pg)
        preprocess_sharded(args.vid_path, env[0], env[1])
        phases.mark("prepass")
        with open(os.path.join(HERE, "config", args.config)) as f:
            main_sharded(json.load(f), args, device, pg, phases)
        launch.finish()
        sys.exit(0)
    os.environ["CUDA_VISIBLE_DEVICES"] = "%d" % args.gpu
    # always run the pre-pass (reference :276-278): it skips the pairs whose files already exist, so a partially
    # written flow folder is completed instead of crashing later in load_input_data_single
    cmd = "%s %s --vid-path %s --gpu %d " % (sys.executable, os.path.join(HERE, "preprocess_optical_flow.py"),
                                             args.vid_path, args.gpu)
    print(cmd)
    if subprocess.call(cmd, shell=True) != 0:
        raise RuntimeError("optical-flow pre-pass failed")
    with open(os.path.join(HERE, "config", args.config)) as f:
        main(json.load(f), args)
