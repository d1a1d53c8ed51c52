"""Pins the stateful TransformNet restatement (tests/convlstm_state_common.py: transformnet_forward_state, on the layers of
oracle/stage2_oracle.py) against the reference's TransformNet (seeded random weights) and freezes transformnet_state.pt:
a 4-frame recurrence at 64x96, each call fed the state the previous one returned (the first one None), and one step
from a random state of magnitude about 3.  Every output is asserted bit-identical to the reference's.  Inputs and
weights are regenerated from seeds (tests/convlstm_state_common.py, tests/nets_common.py); the fixture keeps, per
output, every 17th element and the float64 sum and absolute sum (convlstm_state_common.digest), 80 KB in all.
Replayed by tests/test_convlstm_state_cpu.py.  Build container only (needs /root/reference):
    python tests/golden/make_golden_convlstm_state.py"""
import os
import sys
import types

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, "/root/reference")
for missing in ("imageio", "easydict"):
    sys.modules.setdefault(missing, types.ModuleType(missing))

from src.models.network_local import TransformNet                     # noqa: E402
assert os.path.realpath(sys.modules[TransformNet.__module__].__file__).startswith("/root/reference/"), TransformNet
from nets_common import seeded_weights                                # noqa: E402
from convlstm_state_common import NF, digest, recurrence, recurrence_inputs, transformnet_forward_state  # noqa: E402

WEIGHT_SEED, INPUT_SEED = 23, 24


def same(a, b, what):
    assert torch.equal(a, b), f"{what}: max abs diff {float((a - b).abs().max())}"


def main():
    torch.set_num_threads(1)
    torch.manual_seed(5)
    opts = types.SimpleNamespace(nf=NF, norm="IN", model="TransformNet", blocks=5)
    tn = TransformNet(opts, nc_in=12, nc_out=3).eval()
    shapes = [(k, tuple(v.shape)) for k, v in tn.state_dict().items() if v.dtype.is_floating_point]
    tn.load_state_dict(seeded_weights(shapes, WEIGHT_SEED), strict=False)
    sd = {k: v.detach() for k, v in tn.state_dict().items()}
    xs, x_r, state_r = recurrence_inputs(INPUT_SEED)
    with torch.no_grad():
        ys, state = [], None
        for x in xs:
            ry, state = tn(x, state)
            ys.append(ry)
        oys, ostate = recurrence(sd, xs)
        for t in range(len(xs)):
            same(oys[t], ys[t], f"frame {t} Y")
        same(ostate[0], state[0], "last hidden"); same(ostate[1], state[1], "last cell")
        r_y, (r_h, r_c) = tn(x_r, state_r)
        oy, oh, oc = transformnet_forward_state(sd, x_r, state_r)
        same(oy, r_y, "random-state Y"); same(oh, r_h, "random-state hidden"); same(oc, r_c, "random-state cell")
    print(f"random-state step: |cell| > 2 at {float((r_c.abs() > 2).float().mean()):.0%} of the elements, "
          f"max |cell| {float(r_c.abs().max()):.2f}")
    out = os.path.join(HERE, "transformnet_state.pt")
    torch.save({"shapes": shapes, "seed": WEIGHT_SEED, "input_seed": INPUT_SEED, "nf": NF,
                "ys": [digest(y) for y in ys], "hidden": digest(state[0]), "cell": digest(state[1]),
                "r_y": digest(r_y), "r_hidden": digest(r_h), "r_cell": digest(r_c)}, out)
    print(f"{out} written, {os.path.getsize(out)} bytes")


if __name__ == "__main__":
    main()
