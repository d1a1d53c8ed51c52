"""Stage-1 data helpers with the reference's names (src/models/stage_1/unwrap_utils.py).

`load_input_data_single` is the input producer (reads frames + RAFT flows from disk, CPU, same tensor
layouts as the reference returns); `get_tuples` and `pre_train_mapping` are provided for drop-in use,
the latter running on the fused trainer.  `load_input_data` is the segmentation variant's loader (adds the
bootstrapping masks).  `save_mask_flow` writes the reference's two overview videos with OpenCV.
"""
from pathlib import Path

import numpy as np
import torch
import cv2
from PIL import Image


def _warp_by_flow(img, flow):
    """cv2.remap of `img` at (x + fx, y + fy), bilinear, zeros outside (unwrap_utils.py:17-23)."""
    h, w = flow.shape[:2]
    grid = flow.copy()
    grid[:, :, 0] += np.arange(w)
    grid[:, :, 1] += np.arange(h)[:, None]
    return cv2.remap(img, grid, None, cv2.INTER_LINEAR)


def compute_consistency(flow12, flow21):
    """|flow12 + warp(flow21, flow12)| per pixel (unwrap_utils.py:10-14)."""
    d = flow12 + _warp_by_flow(flow21, flow12)
    return (d[:, :, 0] ** 2 + d[:, :, 1] ** 2) ** .5


def resize_flow(flow, newh, neww):
    """Bilinear resize; note the reference scales x by newh/oldh and y by neww/oldw (unwrap_utils.py:33-38),
    reproduced as is."""
    oldh, oldw = flow.shape[0:2]
    flow = cv2.resize(flow, (neww, newh), interpolation=cv2.INTER_LINEAR)
    flow[:, :, 0] *= newh / oldh
    flow[:, :, 1] *= neww / oldw
    return flow


def load_input_data_single(resy, resx, maximum_number_of_frames, data_folder, use_mask_rcnn_bootstrapping,
                           filter_optical_flow, vid_root, vid_name):
    """Same return tuple as unwrap_utils.py:105-163."""
    flow_dir = vid_root / f'{vid_name}_flow'
    files = sorted(list(data_folder.glob('*.jpg')) + list(data_folder.glob('*.png')))
    T = int(np.minimum(maximum_number_of_frames, len(files)))
    frames = torch.zeros((resy, resx, 3, T))
    dx = torch.zeros_like(frames)
    dy = torch.zeros_like(frames)
    mask_frames = torch.zeros((resy, resx, T))
    flows = torch.zeros((resy, resx, 2, T, 1))
    flows_mask = torch.zeros((resy, resx, T, 1))
    flows_rev = torch.zeros((resy, resx, 2, T, 1))
    flows_rev_mask = torch.zeros((resy, resx, T, 1))
    for i in range(T):
        im = np.array(Image.open(str(files[i]))).astype(np.float64) / 255.
        if im.ndim == 2:
            im = np.tile(im[:, :, None], [1, 1, 3])
        frames[:, :, :, i] = torch.from_numpy(cv2.resize(im[:, :, :3], (resx, resy)))
        dy[:-1, :, :, i] = frames[1:, :, :, i] - frames[:-1, :, :, i]
        dx[:, :-1, :, i] = frames[:, 1:, :, i] - frames[:, :-1, :, i]
    for i in range(T - 1):
        a, b = files[i].name, files[i + 1].name
        f12 = np.load(flow_dir / f'{a}_{b}.npy')
        f21 = np.load(flow_dir / f'{b}_{a}.npy')
        if f12.shape[0] != resy or f12.shape[1] != resx:
            f12 = resize_flow(f12, newh=resy, neww=resx)
            f21 = resize_flow(f21, newh=resy, neww=resx)
        flows[:, :, :, i, 0] = torch.from_numpy(f12)
        flows_rev[:, :, :, i + 1, 0] = torch.from_numpy(f21)
        if filter_optical_flow:
            flows_mask[:, :, i, 0] = torch.from_numpy(compute_consistency(f12, f21) < 1.0)
            flows_rev_mask[:, :, i + 1, 0] = torch.from_numpy(compute_consistency(f21, f12) < 1.0)
        else:
            flows_mask[:, :, i, 0] = 1
            flows_rev_mask[:, :, i + 1, 0] = 1
    return flows_mask, frames, flows_rev_mask, mask_frames, dx, dy, flows_rev, flows


def mask_files(vid_root, vid_name, number_of_frames, clip=None):
    """The matte files of `<vid>_seg` for frames [0, number_of_frames), or for the frames [c0, c1) of `clip`, in sorted
    order.  Refused when the folder holds fewer."""
    mask_dir = Path(vid_root) / f'{vid_name}_seg'
    files = sorted(list(mask_dir.glob('*.jpg')) + list(mask_dir.glob('*.png')))
    c0, c1 = (0, number_of_frames) if clip is None else clip
    if len(files) < c1:
        what = f"{number_of_frames} frames" if clip is None else f"clip_{c0:05d}_{c1:05d} (frames {c0} to {c1 - 1})"
        raise FileNotFoundError(f"{mask_dir}: {len(files)} mask images for {what} — the segmentation "
                                f"variant needs one matte per frame (the reference writes them with "
                                f"src/preprocess_mask_portrait.py / preprocess_mask_rcnn.py)")
    return files[c0:c1]


def load_mask_frames(resy, resx, number_of_frames, vid_root, vid_name, clip=None):
    """(resy, resx, T) bootstrapping masks from `<vid>_seg` (unwrap_utils.py:43,60,67-70).  The reference passes
    cv2.INTER_NEAREST in the position of cv2.resize's `dst` argument, which OpenCV ignores: the masks are resized
    with the default bilinear interpolation, and so they are here.  With `clip` = (c0, c1) (T = c1 - c0): the mattes
    of frames c0..c1-1, as a folder holding only those would give."""
    files = mask_files(vid_root, vid_name, number_of_frames, clip)
    masks = torch.zeros((resy, resx, number_of_frames))
    for i in range(number_of_frames):
        m = np.array(Image.open(str(files[i]))).astype(np.float64) / 255.
        masks[:, :, i] = torch.from_numpy(cv2.resize(m, (resx, resy), interpolation=cv2.INTER_LINEAR))
    return masks


def load_input_data(resy, resx, maximum_number_of_frames, data_folder, use_mask_rcnn_bootstrapping, filter_optical_flow,
                    vid_root, vid_name):
    """Same return tuple as unwrap_utils.py:40-103: `load_input_data_single` plus the masks of `<vid>_seg`."""
    out = list(load_input_data_single(resy, resx, maximum_number_of_frames, data_folder, use_mask_rcnn_bootstrapping,
                                      filter_optical_flow, vid_root, vid_name))
    if use_mask_rcnn_bootstrapping:
        out[3] = load_mask_frames(resy, resx, out[1].shape[3], vid_root, vid_name)
    return tuple(out)


def get_tuples(number_of_frames, video_frames):
    """(3, N) int64 [x; y; t] table (unwrap_utils.py:166-173).  The CUDA path never materialises it: the
    kernels decode n -> (n % W, (n // W) % H, n // (H*W)); this is for callers that want the tensor."""
    H, W = video_frames.shape[0], video_frames.shape[1]
    n = torch.arange(number_of_frames * H * W, dtype=torch.int64)
    return torch.stack((n % W, (n // W) % H, n // (H * W)))


def pre_train_mapping(trainer, frames_num, uv_mapping_scale, resx, resy, larger_dim, device, pretrain_iters=100,
                      which=None):
    """unwrap_utils.py:176-198 on the fused trainer (`b200.atlas.AtlasTrainer`), or on one mapping network of the
    segmentation trainer (`b200.seg.SegTrainer`, which = "mapping1" | "mapping2")."""
    print("pre-training")
    trainer.cfg["uv_mapping_scale"] = uv_mapping_scale
    if which is None:
        trainer.pretrain(frames_num, resy, resx, pretrain_iters)
    else:
        trainer.pretrain(which, frames_num, resy, resx, pretrain_iters)
    return trainer


def save_mask_flow(optical_flows_mask, video_frames, results_folder):
    """unwrap_utils.py:200-231: `filter_flow_<j>.mp4` (frames with the pixels whose forward flow failed the consistency
    check painted red; frames without any valid pixel are skipped) and `input_video.mp4` (the video at the working
    resolution), 10 fps.  Written with OpenCV's mp4 encoder instead of imageio."""
    H, W = int(video_frames.shape[0]), int(video_frames.shape[1])

    def writer(name):
        wr = cv2.VideoWriter(str(results_folder / name) if hasattr(results_folder, "joinpath") else
                             "%s/%s" % (results_folder, name), cv2.VideoWriter_fourcc(*"mp4v"), 10, (W, H))
        if not wr.isOpened():
            raise RuntimeError("OpenCV cannot write mp4 here")
        return wr
    to_bgr = lambda fr: cv2.cvtColor((fr.numpy() * 255).astype(np.uint8), cv2.COLOR_RGB2BGR)
    for j in range(optical_flows_mask.shape[3]):
        wr = writer("filter_flow_%d.mp4" % j)
        for i in range(video_frames.shape[3]):
            m = optical_flows_mask[:, :, i, j]
            if not bool((m == 1).any()):
                continue
            cur = video_frames[:, :, :, i].clone()
            cur[m == 0] = torch.tensor([1.0, 0.0, 0.0])
            wr.write(to_bgr(cur))
        wr.release()
    wr = writer("input_video.mp4")
    for i in range(video_frames.shape[3]):
        wr.write(to_bgr(video_frames[:, :, :, i]))
    wr.release()
