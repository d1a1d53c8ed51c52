"""The dataflows of net_launches_common.py are the reference's networks: driven with a float64 device that evaluates
every layer exactly, they reproduce the oracles to rounding level (1e-12 of the largest output) and the reference's
whole-RAFT fixture within the fp32 bound of test_full_raft_against_reference_fixture.  No GPU, and the reference
project is not read: the oracles and fixtures under tests/golden stand for it."""
import argparse
import os

import numpy as np
import torch

import net_launches_common as NL
from convlstm_state_common import recurrence, recurrence_inputs
from nets_common import seeded_weights
from oracle import flow_oracle as FO
from oracle import stage2_oracle as SO

ROUNDING = 1e-12


def _sd64(sd, prefix=""):
    return {prefix + k: v.double() for k, v in sd.items()}


def _close(what, got, want, tol=ROUNDING):
    err = NL.max_abs_rel(got, want)
    print(f"{what}: max |dataflow - oracle| / max |oracle| = {err:.2e}")
    assert err <= tol, (what, err)


def test_unet_dataflow_is_the_oracle(golden_dir):
    fx = torch.load(os.path.join(golden_dir, "stage2_nets.pt"))
    sd = seeded_weights(fx["unet_shapes"], fx["unet_seed"])
    x = fx["unet_x"].double()
    got = NL.unet(NL.ExactDevice(_sd64(sd, "unet.")), "unet.", x)
    _close("unet", got, SO.unet_forward(_sd64(sd), x))


def test_transformnet_zero_state_dataflow_is_the_oracle(golden_dir):
    fx = torch.load(os.path.join(golden_dir, "stage2_nets.pt"))
    sd = seeded_weights(fx["tn_shapes"], fx["tn_seed"])
    x = fx["tn_x"].double()
    y, (h, c) = NL.transformnet(NL.ExactDevice(_sd64(sd, "tn.")), "tn.", x, None)
    oy, oh, oc = SO.transformnet_forward(_sd64(sd), x)
    for what, a, b in (("Y", y, oy), ("hidden", h, oh), ("cell", c, oc)):
        _close(f"transformnet zero state {what}", a, b)


def test_transformnet_recurrence_dataflow_is_the_oracle(golden_dir):
    """Three frames, each fed the state the previous one returned (the first from the zero state)."""
    fx = torch.load(os.path.join(golden_dir, "transformnet_state.pt"))
    sd = seeded_weights(fx["shapes"], fx["seed"])
    xs, _, _ = recurrence_inputs(fx["input_seed"], frames=3, nf=fx["nf"])
    xs = [x.double() for x in xs]
    ref_ys, ref_state = recurrence(_sd64(sd), xs)
    dev = NL.ExactDevice(_sd64(sd, "tn."))
    state = None
    for t, x in enumerate(xs):
        y, state = NL.transformnet(dev, "tn.", x, state)
        _close(f"transformnet frame {t} Y", y, ref_ys[t])
    _close("transformnet hidden after 3 frames", state[0], ref_state[0])
    _close("transformnet cell after 3 frames", state[1], ref_state[1])


def test_update_block_dataflow_is_the_oracle(golden_dir):
    fx = torch.load(os.path.join(golden_dir, "raft_update.pt"))
    z = np.load(os.path.join(golden_dir, "raft_corr.npz"))
    sd = seeded_weights(fx["shapes"], fx["seed"])
    ins = [fx["net"].double(), fx["inp"].double(), torch.from_numpy(z["lookup"]).double(), fx["flow"].double()]
    got = NL.update_block(NL.ExactDevice(_sd64(sd, "ub.")), "ub.", *ins)
    want = FO.update_block(_sd64(sd), *ins)
    for what, a, b in zip(("net", "mask", "delta"), got, want):
        _close(f"update block {what}", a, b)


def test_whole_raft_dataflow_is_the_reference_fixture(golden_dir):
    """Both encoders (instance norm, batch norm), the all-pairs correlation and lookup of flow_oracle, 3 refinement
    iterations and the convex upsampling, in float64, against the reference's fp32 outputs: 2e-3 of max(|flow|, 1),
    the bound of test_full_raft_against_reference_fixture."""
    from src.models.stage_1.core.raft import RAFT
    from src.models.stage_1.core.utils.utils import coords_grid
    fx = torch.load(os.path.join(golden_dir, "raft_full.pt"))
    model = RAFT(argparse.Namespace(small=False, mixed_precision=False))
    model.load_state_dict(seeded_weights(fx["shapes"], fx["seed"]), strict=False)
    dev = NL.ExactDevice(NL.params_of({"raft.": model}))
    im1, im2 = (2 * (fx[k].double() / 255.0) - 1.0 for k in ("im1", "im2"))
    fmaps = NL.encoder(dev, "raft.fnet.", torch.cat([im1, im2]), "instance")
    cnet = NL.encoder(dev, "raft.cnet.", im1, "batch")
    pyr = FO.corr_pyramid(fmaps[:1], fmaps[1:])
    n, _, h8, w8 = cnet.shape
    coords0 = coords_grid(n, h8, w8).double()
    low, up = NL.refine(dev, "raft.update_block.", cnet, lambda it, c1: FO.corr_lookup(pyr, c1).double(), coords0, 3)
    errs = {}
    for what, a, b in (("flow_low", low, fx["flow_low"]), ("flow_up", up, fx["flow_up"])):
        errs[what] = float((a - b.double()).abs().max()) / max(float(b.abs().max()), 1.0)
    print("whole RAFT dataflow against the reference fixture (relative to max(|flow|, 1)):",
          {k: f"{v:.2e}" for k, v in errs.items()})
    assert max(errs.values()) <= 2e-3, errs
