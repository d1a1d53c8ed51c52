"""Checkpoint + full-video render + PSNR + evaluation artefacts of the reference's `evaluate_model_single`
(src/models/stage_1/evaluate.py:605-793) and of `evaluate_model` (:203-602, segmentation variant).  Reconstruction,
per-pixel maps and PSNR run in libb200deflicker.so; the reconstruction / residual / uv / dashboard videos (:714-779) are
composed with OpenCV (`ArtefactWriter`), tensorboard images go through torch.utils.tensorboard.  The texture-editing
part of the segmentation variant's evaluation (:234-262, :340-600) is interactive-editing tooling and is not provided."""
import os
import time

import cv2
import numpy as np
import torch

from b200 import atlas as A


def _video_writer(path, w, h, fps=10):
    wr = cv2.VideoWriter(path, cv2.VideoWriter_fourcc(*"mp4v"), fps, (int(w), int(h)))
    if not wr.isOpened():
        raise RuntimeError(f"cannot open {path} for writing (OpenCV was built without an mp4 encoder)")
    return wr


def _heat(a, vmin, vmax):
    """Scalar map -> BGR heat image (the dashboards' imshow(vmin, vmax) panels, evaluate.py:745-760)."""
    g = np.clip((np.asarray(a, np.float64) - vmin) / (vmax - vmin), 0, 1)
    return cv2.applyColorMap((g * 255).astype(np.uint8), cv2.COLORMAP_VIRIDIS)


def _panel(img_bgr, title):
    out = cv2.copyMakeBorder(img_bgr, 22, 0, 0, 0, cv2.BORDER_CONSTANT, value=(255, 255, 255))
    cv2.putText(out, title, (4, 16), cv2.FONT_HERSHEY_SIMPLEX, 0.5, (0, 0, 0), 1, cv2.LINE_AA)
    return out


def artefact_images(frame, recon, uv, rigidity, flow_error):
    """The reconstruction, residual, uv and dashboard BGR uint8 images of one frame (ArtefactWriter.add's inputs)."""
    bgr = lambda a: cv2.cvtColor((np.clip(a, 0, 1) * 255).astype(np.uint8), cv2.COLOR_RGB2BGR)
    res = frame - recon
    uv_img = np.zeros(recon.shape, np.float64)
    uv_img[:, :, :2] = np.clip(uv * 0.5 + 0.5, 0, 1)                                   # normalize_uv_images, :193-200
    err = (res.astype(np.float64) ** 2).sum(-1)                                        # :702
    top = np.concatenate([_panel(bgr(recon), "video_reconstruction"), _panel(bgr(frame), "original_video"),
                          _panel(_heat(err, 0.0, 0.2), "RGB error")], axis=1)
    bot = np.concatenate([_panel(_heat(flow_error, 0.0, 2.0), "flow_loss1"),
                          _panel(_heat(rigidity, 2.8, 50.0), "rigidity_loss1"), _panel(bgr(uv_img), "uv")], axis=1)
    return [bgr(recon), bgr(res + 0.5), bgr(uv_img), np.concatenate([top, bot], axis=0)]      # :726 for the residual


class ArtefactWriter:
    """The per-iteration evaluation output of evaluate.py:714-793: `reconstruction_<vid>.mp4`, `residuals_<vid>.mp4`,
    `uv_1_<vid>.mp4` and the `global_info_<vid>.mp4` dashboard (reconstruction | original | RGB error | flow error |
    rigidity, with the reference's colour ranges), written with OpenCV (imageio / matplotlib are not needed)."""

    def __init__(self, folder, vid_name, resx, resy):
        self.names = ("reconstruction", "residuals", "uv_1", "global_info")
        self.w = {k: _video_writer(os.path.join(folder, f"{k}_{vid_name}.mp4"), resx, resy) for k in self.names[:3]}
        self.w["global_info"] = _video_writer(os.path.join(folder, f"global_info_{vid_name}.mp4"), 3 * resx, 2 * (resy + 22))

    def add(self, frame, recon, uv, rigidity, flow_error):
        """frame, recon: (H, W, 3) fp32 RGB in [0, 1]; uv (H, W, 2); rigidity, flow_error (H, W) — numpy arrays."""
        self.write(artefact_images(frame, recon, uv, rigidity, flow_error))

    def write(self, images):
        """The four BGR images of one frame (artefact_images), in the order of `names`."""
        for k, img in zip(self.names, images):
            self.w[k].write(img)

    def close(self):
        for w in self.w.values():
            w.release()


def evaluate_model_single(trainer, resx, resy, number_of_frames, video_frames, results_folder, iteration,
                          vid_name=None, save_checkpoint=True, artefacts=False, writer=None, output_folder=None,
                          frame_offset=0, write_frames=None):
    """Frame f's reconstruction goes to `<output_folder>/%05d.png % (frame_offset + f)` (default `<results_folder>/output`,
    offset 0): a clip of a longer video writes its frames where they lie in the video.  With `write_frames` (a
    collection of frames f) only those frames' files are written; everything else, PSNR included, covers every frame."""
    output_folder = os.path.join(results_folder, "output") if output_folder is None else output_folder
    os.makedirs(os.path.join(results_folder, '%06d' % iteration), exist_ok=True)
    os.makedirs(output_folder, exist_ok=True)
    if save_checkpoint:      # evaluate.py:616-622 — same file name and keys
        torch.save(trainer.checkpoint(iteration), '%s/checkpoint' % results_folder)
    psnrs = np.zeros((number_of_frames, 1))
    art = ArtefactWriter(os.path.join(results_folder, '%06d' % iteration), vid_name or "video", resx, resy) if artefacts else None
    ends = {}
    for f in range(number_of_frames):
        img, u8 = trainer.render_frame(f, int(resy), int(resx), number_of_frames, want_u8=True)
        if write_frames is None or f in write_frames:
            cv2.imwrite(os.path.join(output_folder, '%05d.png' % (frame_offset + f)),
                        cv2.cvtColor(u8.cpu().numpy(), cv2.COLOR_RGB2BGR))   # evaluate.py:732-733
        psnrs[f] = A.psnr(video_frames[:, :, :, f], img.cpu())               # :740-743
        if art is not None:                                                  # :668-779, maps computed on the device
            uv, rig, flow = trainer.eval_maps(f)
            art.add(video_frames[:, :, :, f].numpy(), img.cpu().numpy(), uv.cpu().numpy(), rig.cpu().numpy(),
                    flow.cpu().numpy())
        if f in (0, number_of_frames - 1):
            ends[f] = img.cpu().numpy()
    if art is not None:
        art.close()
    if writer is not None and save_checkpoint:                               # tensorboard images, :784-793
        writer.add_image("Train/recon_frame_0", ends[0], iteration, dataformats='HWC')
        writer.add_image("Train/recon_frame_end", ends[number_of_frames - 1], iteration, dataformats='HWC')
    open(os.path.join(results_folder, '%06d' % iteration, "PSNR_%f" % psnrs.mean()), "w").close()   # :782
    print("PSNR: %f" % psnrs.mean())
    return float(psnrs.mean())


def evaluate_model(trainer, resx, resy, number_of_frames, video_frames, results_folder, iteration, mask_frames=None,
                   vid_name=None, save_checkpoint=True, output_folder=None, frame_offset=0, write_frames=None):
    """Segmentation variant (evaluate.py:203-602): checkpoint with the reference's keys (:216-233), the composite
    reconstruction (:293-335) written to `output/`, the alpha mattes to `<iteration>/alpha/`, PSNR.  Texture editing,
    atlas dumps and per-pixel loss videos are visualisation (out of scope).  `output_folder`, `frame_offset` and
    `write_frames` as in evaluate_model_single; the alpha mattes keep the clip's own frame numbers."""
    output_folder = os.path.join(results_folder, "output") if output_folder is None else output_folder
    folder = os.path.join(results_folder, '%06d' % iteration)
    os.makedirs(os.path.join(folder, "alpha"), exist_ok=True)
    os.makedirs(output_folder, exist_ok=True)
    if save_checkpoint:
        ck = trainer.checkpoint(iteration)
        torch.save(ck, '%s/checkpoint' % results_folder)
        torch.save(ck, '%s/checkpoint' % folder)
    psnrs = np.zeros((number_of_frames, 1))
    for f in range(number_of_frames):
        img, alpha, u8 = trainer.render_frame(f, int(resy), int(resx), number_of_frames, want_u8=True)
        if write_frames is None or f in write_frames:
            cv2.imwrite(os.path.join(output_folder, '%05d.png' % (frame_offset + f)),
                        cv2.cvtColor(u8.cpu().numpy(), cv2.COLOR_RGB2BGR))
        cv2.imwrite(os.path.join(folder, 'alpha', '%05d.png' % f), (alpha.cpu().numpy() * 255).astype(np.uint8))
        psnrs[f] = A.psnr(video_frames[:, :, :, f], img.cpu())
    open(os.path.join(folder, "PSNR_%f" % psnrs.mean()), "w").close()
    print("PSNR: %f" % psnrs.mean())
    return float(psnrs.mean())


# ---------------------------------------------------------------------------------------------------------------------
# Frame-sharded evaluation: every rank of a process group renders and scores the frames of its block (trainer.video),
# rank 0 assembles what covers the whole video.

def _pack(images):
    return torch.from_numpy(np.concatenate([np.ascontiguousarray(im).reshape(-1) for im in images]))


def _unpack(buf, resx, resy):
    shapes = [(resy, resx, 3)] * 3 + [(2 * (resy + 22), 3 * resx, 3)]
    out, o = [], 0
    a = buf.numpy()
    for s in shapes:
        n = int(np.prod(s))
        out.append(a[o:o + n].reshape(s))
        o += n
    return out


def artefact_payload_bytes(resx, resy):
    """Bytes of one frame's packed artefact images (reconstruction, residuals, uv, dashboard)."""
    return 3 * resy * resx * 3 + 2 * (resy + 22) * 3 * resx * 3


def evaluate_block_single(trainer, resx, resy, number_of_frames, results_folder, artefacts=False, write_frames=None):
    """The frames of trainer.video's resident block: writes `output/%05d.png` (of the frames in `write_frames` only,
    when given), returns (per-frame PSNR, packed artefact images per frame or []).  The PSNR's squared error is summed on the device against the resident records
    (b200_frame_sse), and the original frame of the artefact images is read from them too."""
    video = trainer.video
    psnrs, payloads = [], []
    for f in range(video.t_begin, video.t_end):
        img, u8 = trainer.render_frame(f, int(resy), int(resx), number_of_frames, want_u8=True)
        if write_frames is None or f in write_frames:
            cv2.imwrite(os.path.join(results_folder, 'output', '%05d.png' % f),
                        cv2.cvtColor(u8.cpu().numpy(), cv2.COLOR_RGB2BGR))
        psnrs.append(A.psnr_device(video, f, img))
        if artefacts:
            uv, rig, flow = trainer.eval_maps(f)
            payloads.append(_pack(artefact_images(video.frame_rgb(f).cpu().numpy(), img.cpu().numpy(), uv.cpu().numpy(),
                                                  rig.cpu().numpy(), flow.cpu().numpy())))
    return psnrs, payloads


def write_evaluation_single(trainer, resx, resy, number_of_frames, results_folder, iteration, psnrs, vid_name=None,
                            artefacts=None, writer=None, save_checkpoint=True):
    """Rank 0's part: the four evaluation videos from `artefacts` (packed images of every frame in frame order, or
    None), the two tensorboard images (frames 0 and T-1, rendered here: they need parameters only) and the PSNR marker
    of the merged per-frame `psnrs`.  Returns the mean PSNR."""
    folder = os.path.join(results_folder, '%06d' % iteration)
    if artefacts is not None:
        art = ArtefactWriter(folder, vid_name or "video", resx, resy)
        for buf in artefacts:
            art.write(_unpack(buf, resx, resy))
        art.close()
    if writer is not None and save_checkpoint:
        for f, tag in ((0, "Train/recon_frame_0"), (number_of_frames - 1, "Train/recon_frame_end")):
            img = trainer.render_frame(f, int(resy), int(resx), number_of_frames)
            writer.add_image(tag, img.cpu().numpy(), iteration, dataformats='HWC')
    mean = float(np.mean(psnrs))
    open(os.path.join(folder, "PSNR_%f" % mean), "w").close()
    print("PSNR: %f" % mean)
    return mean


def evaluate_model_single_sharded(trainer, resx, resy, number_of_frames, results_folder, iteration, vid_name=None,
                                  save_checkpoint=True, artefacts=False, writer=None, process_group=None,
                                  write_frames=None):
    """evaluate_model_single over a process group whose ranks hold contiguous frame blocks (collective): the same
    checkpoint (written by rank 0 after the collective optimizer_state_dict), frames, marker and videos."""
    import torch.distributed as dist
    from b200 import launch
    pg = process_group
    rank, world = dist.get_rank(pg), dist.get_world_size(pg)
    os.makedirs(os.path.join(results_folder, '%06d' % iteration), exist_ok=True)
    os.makedirs(os.path.join(results_folder, "output"), exist_ok=True)
    if save_checkpoint:
        ck = trainer.checkpoint(iteration)        # collective: every rank gathers the Adam moments
        if rank == 0:
            torch.save(ck, '%s/checkpoint' % results_folder)
    psnrs, payloads = evaluate_block_single(trainer, resx, resy, number_of_frames, results_folder, artefacts,
                                            write_frames)
    merged = launch.gather_frame_values(psnrs, pg)
    received = []
    if artefacts:
        counts = [b - a for a, b in (A.frame_range(r, world, number_of_frames) for r in range(world))]
        launch.collect_on_root(payloads, counts, artefact_payload_bytes(resx, resy), received.append, trainer.device, pg)
    mean = float(np.mean(merged))
    if rank == 0:
        mean = write_evaluation_single(trainer, resx, resy, number_of_frames, results_folder, iteration, merged, vid_name,
                                       received if artefacts else None, writer, save_checkpoint)
    dist.barrier(pg)
    return mean


def evaluate_block_seg(trainer, resx, resy, number_of_frames, results_folder, iteration, write_frames=None):
    """Segmentation variant: the frames of trainer.video's block — `output/%05d.png` (of the frames in `write_frames`
    only, when given), `<iteration>/alpha/%05d.png` — and their PSNR (device squared error against the resident
    records)."""
    folder = os.path.join(results_folder, '%06d' % iteration)
    video = trainer.video
    psnrs = []
    for f in range(video.t_begin, video.t_end):
        img, alpha, u8 = trainer.render_frame(f, int(resy), int(resx), number_of_frames, want_u8=True)
        if write_frames is None or f in write_frames:
            cv2.imwrite(os.path.join(results_folder, 'output', '%05d.png' % f),
                        cv2.cvtColor(u8.cpu().numpy(), cv2.COLOR_RGB2BGR))
        cv2.imwrite(os.path.join(folder, 'alpha', '%05d.png' % f), (alpha.cpu().numpy() * 255).astype(np.uint8))
        psnrs.append(A.psnr_device(video, f, img))
    return psnrs


def evaluate_model_sharded(trainer, resx, resy, number_of_frames, results_folder, iteration, vid_name=None,
                           save_checkpoint=True, process_group=None, write_frames=None):
    """evaluate_model over a process group whose ranks hold contiguous frame blocks (collective)."""
    import torch.distributed as dist
    from b200 import launch
    pg = process_group
    rank = dist.get_rank(pg)
    folder = os.path.join(results_folder, '%06d' % iteration)
    os.makedirs(os.path.join(folder, "alpha"), exist_ok=True)
    os.makedirs(os.path.join(results_folder, "output"), exist_ok=True)
    if save_checkpoint:
        ck = trainer.checkpoint(iteration)        # collective: every rank gathers the Adam moments
        if rank == 0:
            torch.save(ck, '%s/checkpoint' % results_folder)
            torch.save(ck, '%s/checkpoint' % folder)
    merged = launch.gather_frame_values(evaluate_block_seg(trainer, resx, resy, number_of_frames, results_folder, iteration,
                                                           write_frames), pg)
    mean = float(np.mean(merged))
    if rank == 0:
        open(os.path.join(folder, "PSNR_%f" % mean), "w").close()
        print("PSNR: %f" % mean)
    dist.barrier(pg)
    return mean


# ---------------------------------------------------------------------------------------------------------------------
# Seams of overlapping clips (--clips --clip_overlap V): the V frames two consecutive clips share are a cross-fade of
# the two atlases' renders, so the jump between the atlases is spread over V + 1 frame steps (DESIGN §5).

def _render_rgb(trainer, f, H, W, T):
    out = trainer.render_frame(f, H, W, T)
    return out[0] if isinstance(out, tuple) else out          # SegTrainer: (rgb, alpha)


def stitch_seams(plan, make_trainer, stage_folder, resx, resy, rank=0, world=1):
    """Writes the shared frames of the seams of `plan` (b200.atlas.clip_plan with an overlap) that rank `rank` of
    `world` owns (seam k for k = rank mod world, atlas.rank_seams) to `<stage_folder>/output/%05d.png`.  Frame a + j
    of seam k, [a, b) = atlas.clip_seams(plan)[k], is b200_blend_frames of clip k's and clip k+1's renders, each at
    its own clip-local frame index and frame count, with the weight w_j = (j + 1) / (V + 1) of atlas.seam_weights on
    clip k+1, quantised and written (RGB -> BGR) as the evaluation writes a frame.  `make_trainer(path)` builds a
    render-only trainer of the variant from a clip's `checkpoint` file: the parameters of the clip's last
    evaluation, which wrote its other frames.  Every checkpoint must exist, so ranks call this after the clips'
    barrier; when a clip has none (no evaluation ran, and no frame was written) nothing is stitched.  Returns the
    number of frames written."""
    seams = A.clip_seams(plan)
    checkpoints = [os.path.join(str(stage_folder), A.clip_name(c), "checkpoint") for c in plan]
    missing = [p for p in checkpoints if not os.path.exists(p)]
    if missing:
        if rank == 0:
            print("stitch: no evaluation wrote %s; nothing was stitched" % missing[0], flush=True)
        return 0
    output_folder = os.path.join(str(stage_folder), "output")
    os.makedirs(output_folder, exist_ok=True)
    H, W = int(resy), int(resx)
    written, start = 0, time.perf_counter()
    for k in A.rank_seams(seams, rank, world):
        (a, b), (l0, l1), (r0, r1) = seams[k], plan[k], plan[k + 1]
        if b <= a:
            continue
        left, right = make_trainer(checkpoints[k]), make_trainer(checkpoints[k + 1])
        for j, w in enumerate(A.seam_weights(b - a)):
            t = a + j
            _, u8 = A.blend_frames(_render_rgb(left, t - l0, H, W, l1 - l0), _render_rgb(right, t - r0, H, W, r1 - r0), w,
                                   want_out=False, want_u8=True)
            cv2.imwrite(os.path.join(output_folder, '%05d.png' % t), cv2.cvtColor(u8.cpu().numpy(), cv2.COLOR_RGB2BGR))
            written += 1
        left.release()
        right.release()
    print("stitch: rank %d wrote %d frames of %d seams in %.2f s" % (rank, written, len(A.rank_seams(seams, rank, world)),
                                                                   time.perf_counter() - start), flush=True)
    return written
