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
the clips spread over the ranks under torchrun; see `driver.fit_clips`.  With --clip_overlap V consecutive clips share
V frames, which are written once every clip is fitted as a cross-fade of the two atlases' renders; see `driver.stitch`.

The mattes of `<root>/<NAME>_seg/` are an input: the reference produces them with third-party models (CarveKit /
detectron2 Mask-RCNN, src/preprocess_mask_*.py) that this repository does not ship; the script stops with a clear
message when they are missing.
"""
import glob
import os
import sys
from pathlib import Path

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from b200 import seg as SG     # noqa: E402
from src.models.stage_1 import driver  # noqa: E402
from src.models.stage_1.evaluate import evaluate_model, evaluate_model_sharded  # noqa: E402
from src.models.stage_1.unwrap_utils import load_mask_frames, mask_files  # noqa: E402


class Seg(driver.Variant):
    """The two-layer atlas of (mapping1, mapping2, alpha, atlas), bootstrapped by the mattes of `<NAME>_seg/`; both
    mappings pre-trained; evaluations write the composite frames and the alpha mattes."""

    pretrain = {"mapping1": "pretrain_mapping1", "mapping2": "pretrain_mapping2"}

    def trainer(self, video, config, vid_path=None, clip=None, **kw):
        mask = None
        if video is not None:        # the mattes of the video's resident frames
            folder = Path(vid_path)
            mattes = load_mask_frames(video.H, video.W, video.T, folder.parent, folder.name, clip=clip)
            mask = SG.pack_mask_frames(mattes, kw["device"], video.t_begin, video.t_end)
        return SG.SegTrainer(video, mask, config, **kw)

    def evaluate(self, trainer, resx, resy, T, frames, folder, it, vid_name, artefacts, writer, **output):
        evaluate_model(trainer, resx, resy, T, frames, folder, it, vid_name=vid_name, **output)

    def evaluate_sharded(self, trainer, resx, resy, T, folder, it, vid_name, artefacts, writer, pg):
        evaluate_model_sharded(trainer, resx, resy, T, folder, it, vid_name, process_group=pg)

    def check_inputs(self, args):
        seg_dir = args.vid_path.rstrip("/") + "_seg"
        if not glob.glob(os.path.join(seg_dir, "*g")):
            raise FileNotFoundError(f"{seg_dir} holds no mattes: produce them with the reference's mask pre-pass "
                                    f"(class '{args.class_name}') or any segmentation tool, one image per frame")

    def check_clips(self, vid_path, clips):
        check_clip_mattes(vid_path, clips)


VARIANT = Seg()


def check_clip_mattes(vid_path, clips):
    """Refuse, naming the first clip concerned, a matte folder that holds fewer mattes than the video has frames."""
    data_folder = Path(vid_path)
    for clip in clips:
        mask_files(data_folder.parent, data_folder.name, clip[1] - clip[0], clip)


def flags(parser):
    parser.add_argument('--down', type=int, default=1)
    parser.add_argument('--gpu', type=str, default="0")
    parser.add_argument('--class_name', type=str, default="portrait")


if __name__ == "__main__":
    driver.run(VARIANT, driver.parse_args(flags))
