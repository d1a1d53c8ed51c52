"""Pipeline driver with the reference's CLI (test.py:4-42): split the video into frames, run stage 1
(neural atlas) and, when available, stage 2.  ffmpeg is used when installed, otherwise OpenCV."""
import argparse
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))

parser = argparse.ArgumentParser()
parser.add_argument('--video_name', type=str, default=None)
parser.add_argument('--video_frame_folder', type=str, default=None)
parser.add_argument('--fps', type=int, default=10)
parser.add_argument('--gpu', type=int, default=0)
parser.add_argument('--gpus', type=int, default=1,
                    help="run the flow pre-pass, stage 1 and stage 2 on this many GPUs of the node")
parser.add_argument('--class_name', type=str, default=None)
parser.add_argument('--clips', action='store_true',
                    help="stage 1 fits a video longer than maximum_number_of_frames as clips, one atlas each")
parser.add_argument('--clip_overlap', type=int, default=0,
                    help="with --clips: consecutive clips share this many frames, written as a cross-fade of the two "
                         "atlases' renders")
parser.add_argument('--evaluate_flicker', action='store_true',
                    help="after stage 2, score the warping error of the input and of every output (results/<name>/flicker.json)")
parser.add_argument('--fidelity', action='store_true',
                    help="with --evaluate_flicker: also score SSIM and PSNR of every output against the input or "
                         "--reference (results/<name>/fidelity.json)")
parser.add_argument('--reference', type=str, default=None,
                    help="with --fidelity: the folder of reference frames, for example a video's clean frames")
parser.add_argument('--ckpt_filter', type=str, default="./pretrained_weights/neural_filter.pth")
parser.add_argument('--ckpt_local', type=str, default="./pretrained_weights/local_refinement_net.pth")


def split_video(path, out_dir, fps):
    os.makedirs(out_dir, exist_ok=True)
    if shutil.which("ffmpeg"):
        subprocess.check_call(["ffmpeg", "-y", "-i", path, "-vf", f"fps={fps}", "-start_number", "0",
                               os.path.join(out_dir, "%05d.png")])
        return
    import cv2
    cap = cv2.VideoCapture(path)
    src_fps = cap.get(cv2.CAP_PROP_FPS) or fps
    step, t_next, idx, k = src_fps / fps, 0.0, 0, 0
    while True:
        ok, frame = cap.read()
        if not ok:
            break
        if idx + 1e-6 >= t_next:
            cv2.imwrite(os.path.join(out_dir, "%05d.png" % k), frame)
            k += 1
            t_next += step
        idx += 1


if __name__ == "__main__":
    args = parser.parse_args()
    if args.clip_overlap != 0 and not args.clips:
        parser.error("--clip_overlap is only meaningful with --clips")
    if args.clip_overlap < 0:
        parser.error("--clip_overlap must be >= 0")
    if args.fidelity and not args.evaluate_flicker:
        parser.error("--fidelity is only meaningful with --evaluate_flicker")
    if args.reference is not None and not args.fidelity:
        parser.error("--reference is only meaningful with --fidelity")
    # The reference (test.py:17-31) always works on ./data/test/<name>: a video is split into that folder, a frame
    # folder is moved there.  Stage 1 (--root data/test/) and stage 2 (hard-coded ./data/test/<name>) both read it.
    if args.video_name is not None:
        name = os.path.basename(args.video_name)[:-4]
        frames_dir = os.path.join(".", "data", "test", name)
        split_video(args.video_name, frames_dir, args.fps)
    else:
        name = os.path.basename(os.path.normpath(args.video_frame_folder))
        frames_dir = os.path.join(".", "data", "test", name)
        if os.path.isdir(frames_dir):
            print("input folder {} exist".format(frames_dir))
        else:
            os.makedirs(os.path.dirname(frames_dir), exist_ok=True)
            print("mv {} {}".format(args.video_frame_folder, frames_dir))
            shutil.move(args.video_frame_folder, frames_dir)
    if args.class_name is None:
        stage1 = [sys.executable, os.path.join(HERE, "src", "stage1_neural_atlas.py"), "--vid_name", name,
                  "--gpu", str(args.gpu)]
    else:
        # the two-layer variant (reference test.py:39); it needs the mattes of data/test/<name>_seg
        stage1 = [sys.executable, os.path.join(HERE, "src", "stage1_neural_atlas_seg.py"), "--vid_name", name,
                  "--class_name", args.class_name, "--gpu", str(args.gpu)]
    stage2 = [sys.executable, os.path.join(HERE, "src", "neural_filter_and_refinement.py"), "--video_name", name,
              "--fps", str(args.fps), "--ckpt_filter", args.ckpt_filter, "--ckpt_local", args.ckpt_local]
    if args.gpus > 1:
        # both stages re-run themselves under torchrun on cuda:0..N-1
        stage1 += ["--gpus", str(args.gpus)]
        stage2 += ["--gpus", str(args.gpus)]
    if args.clips:
        # stage 2 runs over the whole video's output frames as it is
        stage1 += ["--clips"]
    if args.clip_overlap > 0:
        stage1 += ["--clip_overlap", str(args.clip_overlap)]
    rc = subprocess.call(stage1)
    if rc != 0:
        sys.exit(rc)
    rc = subprocess.call(stage2)
    if rc != 0 or not args.evaluate_flicker:
        sys.exit(rc)
    flicker = [sys.executable, os.path.join(HERE, "src", "evaluate_flicker.py"), "--video_name", name, "--gpu", str(args.gpu)]
    if args.gpus > 1:
        flicker += ["--gpus", str(args.gpus)]
    if args.clips:
        flicker += ["--clips"]
    if args.clip_overlap > 0:
        flicker += ["--clip_overlap", str(args.clip_overlap)]
    if args.fidelity:
        flicker += ["--fidelity"]
    if args.reference is not None:
        # the script runs from this directory too, so a relative folder means the same
        flicker += ["--reference", args.reference]
    sys.exit(subprocess.call(flicker))
