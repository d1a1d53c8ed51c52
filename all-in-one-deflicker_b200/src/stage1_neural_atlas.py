"""Stage 1 — fit the neural atlas of one video.  Same CLI, config keys, on-disk inputs and outputs as
the reference script (src/stage1_neural_atlas.py:257-281); the optimisation loop itself
(:151-231) runs as one replayed CUDA graph per iteration in libb200deflicker.so.

    python src/stage1_neural_atlas.py --vid_name NAME [--config config_flow_100.json] [--root data/test/]
                                      [--down 4] [--gpu 0] [--gpus 1] [--clips [--clip_overlap V]]

With --gpus N > 1 the script re-runs itself under `python -m torch.distributed.run --nproc-per-node N`; under torchrun
(any world size) every rank computes a block of the flow pairs, holds a block of the frames and evaluates those.

With --clips a video longer than maximum_number_of_frames is fitted as clips (b200.atlas.clip_plan), one atlas each,
the clips spread over the ranks under torchrun; see `driver.fit_clips`.  With --clip_overlap V consecutive clips share
V frames, which are written once every clip is fitted as a cross-fade of the two atlases' renders; see `driver.stitch`.
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from b200 import atlas as A    # noqa: E402
from src.models.stage_1 import driver  # noqa: E402
from src.models.stage_1.evaluate import evaluate_model_single, evaluate_model_single_sharded  # noqa: E402


class Atlas(driver.Variant):
    """The atlas of (mapping, atlas), the mapping pre-trained, evaluations with the reference's artefacts."""

    pretrain = {None: "pretrain_mapping1"}

    def trainer(self, video, config, vid_path=None, clip=None, **kw):
        return A.AtlasTrainer(video, config, **kw)

    def artefacts(self, args):
        return not args.no_artefacts

    def evaluate(self, trainer, resx, resy, T, frames, folder, it, vid_name, artefacts, writer, **output):
        evaluate_model_single(trainer, resx, resy, T, frames, folder, it, vid_name, artefacts=artefacts, writer=writer,
                              **output)

    def evaluate_sharded(self, trainer, resx, resy, T, folder, it, vid_name, artefacts, writer, pg):
        evaluate_model_single_sharded(trainer, resx, resy, T, folder, it, vid_name, artefacts=artefacts, writer=writer,
                                      process_group=pg)


VARIANT = Atlas()


def flags(parser):
    parser.add_argument('--down', type=int, default=4)
    parser.add_argument('--gpu', type=int, default=0)
    parser.add_argument('--no_artefacts', action='store_true',
                        help="skip the evaluation videos / tensorboard log (checkpoint, output frames and PSNR only)")


if __name__ == "__main__":
    driver.run(VARIANT, driver.parse_args(flags))
