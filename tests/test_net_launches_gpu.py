"""Stage 2's networks and RAFT's encoders and update block, launch by launch at the benchmark geometry, on both
convolution paths: every launch against float64 on its own operands, every operand against the reference's dataflow
(net_launches_common.py states the checks and their bounds).

- Stage 2 at 1088 x 1920 (n = 1): UNet, and TransformNet on three smooth frames that differ slightly from one to the
  next: the zero state, then two frames on the carried state (a state one frame stale fails the operand check).
- RAFT as `forward_sequence` runs a window of K + 1 = 3 frames of 1080 x 1920: fnet (instance norm) and cnet (batch
  norm folded into the convolutions) on the three frames at once, then two refinement iterations without the CUDA
  graph on the 2K = 4 flows.  Features are 135 x 240 (odd height); the encoders normalise planes of 540 x 960 =
  518 400 pixels.  The correlation, pinned elsewhere, is the on-the-fly one (`alternate_corr`), which needs no
  all-pairs volume; its lookups are taken as given.
- Each test runs a second geometry in the same process, in the order small, benchmark, small: 480 x 854 content, stage 2
  padded to 480 x 864 and RAFT features of 60 x 107.  The operand checks are repeated every time, so that no chained
  buffer, weight image, merged or folded weight cached for one geometry leaks into another.

Weights are `nets_common.seeded_weights` with the fixtures' seeds.  Launches are recorded and checked one network
forward (one TransformNet frame) at a time, then dropped.  Each test prints the largest error / bound per network and
path, its wall time and its peak device memory."""
import argparse
import os
import time
import types

import pytest
import torch
import torch.nn.functional as F

import net_launches_common as NL
from b200 import nn as K
from csrc_build import ensure_built
from nets_common import seeded_weights

pytestmark = pytest.mark.gpu
DEV = "cuda"
GEOMETRIES = [(480, 854), (1080, 1920), (480, 854)]


@pytest.fixture(scope="module", autouse=True)
def _built():
    ensure_built()


@pytest.fixture
def precision(request):
    prev = K.set_conv_precision(request.param)
    yield request.param
    K.set_conv_precision(prev)


def _pad32(n):
    return -(-n // 32) * 32


def _smooth(g, c, h, w, cell=24):
    """Smooth values in [0, 1): bilinear interpolation of a coarse random grid."""
    t = torch.rand(1, c, h // cell + 2, w // cell + 2, generator=g)
    return F.interpolate(t, size=(h, w), mode="bilinear", align_corners=False).contiguous()


def _report(what, ratios, t0):
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    print(f"{what}: largest error / bound " + ", ".join(f"{k} {v:.3f}" for k, v in sorted(ratios.items())) +
          f"; wall {time.perf_counter() - t0:.1f} s, peak device memory {peak:.2f} GiB")


def _check(rec, params, label, ratios, flow):
    chk = NL.LaunchChecker(rec, params, label, ratios)
    out = flow(chk)
    chk.finish()
    return out


@pytest.mark.parametrize("precision", ["tc", "fp32"], indirect=True)
def test_stage2_networks_launch_by_launch(golden_dir, precision):
    from src.models.network_filter import UNet
    from src.models.network_local import TransformNet
    t0 = time.perf_counter()
    torch.cuda.reset_peak_memory_stats()
    fx = torch.load(os.path.join(golden_dir, "stage2_nets.pt"))
    unet = UNet(in_channels=6, out_channels=3, init_features=32)
    unet.load_state_dict(seeded_weights(fx["unet_shapes"], fx["unet_seed"]))
    unet = unet.to(DEV).eval()
    fs = torch.load(os.path.join(golden_dir, "transformnet_state.pt"))
    tn = TransformNet(types.SimpleNamespace(nf=fs["nf"], norm="IN", model="TransformNet", blocks=5), nc_in=12, nc_out=3)
    tn.load_state_dict(seeded_weights(fs["shapes"], fs["seed"]), strict=False)
    tn = tn.to(DEV).eval()
    up, tp = NL.params_of({"unet.": unet}), NL.params_of({"tn.": tn})
    ratios = {}
    for gi, (h, w) in enumerate(GEOMETRIES):
        hp, wp = _pad32(h), _pad32(w)
        g = torch.Generator().manual_seed(hp * 7 + gi)
        x = _smooth(g, 6, hp, wp).to(DEV)
        with NL.Recorder({"unet.": unet}) as rec:
            y = unet(x)
        got = _check(rec, up, f"unet[{precision}]", ratios, lambda d: NL.unet(d, "unet.", x))
        assert torch.equal(got, y)
        del rec, got, y
        base, drift = _smooth(g, 12, hp, wp).to(DEV), _smooth(g, 12, hp, wp).to(DEV) - 0.5
        state, flow_state = None, None
        for t in range(3):
            xt = (base + 0.03 * t * drift).contiguous()
            with NL.Recorder({"tn.": tn}) as rec:
                y, state = tn(xt, state)
            got, flow_state = _check(rec, tp, f"transformnet[{precision}]", ratios,
                                     lambda d: NL.transformnet(d, "tn.", xt, flow_state))
            assert torch.equal(got, y) and torch.equal(flow_state[0], state[0]) and torch.equal(flow_state[1], state[1])
            del rec
    _report(f"stage 2 [{precision}]", ratios, t0)


@pytest.mark.parametrize("precision", ["tc", "fp32"], indirect=True)
def test_raft_launches_as_forward_sequence_runs_a_window(golden_dir, precision):
    from src.models.stage_1.core.raft import RAFT
    from src.models.stage_1.core.utils.utils import coords_grid
    t0 = time.perf_counter()
    torch.cuda.reset_peak_memory_stats()
    fx = torch.load(os.path.join(golden_dir, "raft_full.pt"))
    model = RAFT(argparse.Namespace(small=False, mixed_precision=False, cuda_graph=False, alternate_corr=True))
    model.load_state_dict(seeded_weights(fx["shapes"], fx["seed"]), strict=False)
    model = model.to(DEV).eval()
    params = NL.params_of({"raft.": model})
    ratios = {}
    iters = 2
    for gi, (h, w) in enumerate(GEOMETRIES):
        g = torch.Generator().manual_seed(h * 5 + gi)
        base = _smooth(g, 3, h, w, cell=40)
        frames = torch.cat([torch.roll(base, shifts=(k, 2 * k), dims=(2, 3)) for k in range(3)]) * 255.0
        x = (2 * (frames.to(DEV) / 255.0) - 1.0).contiguous()      # forward_sequence's normalisation
        outs = {}
        for enc, norm in (("fnet", "instance"), ("cnet", "batch")):
            with NL.Recorder({"raft.": model}) as rec:
                y = getattr(model, enc)(x)
            outs[enc] = _check(rec, params, f"raft.{enc}[{precision}]", ratios,
                               lambda d: NL.encoder(d, f"raft.{enc}.", x, norm))
            assert torch.equal(outs[enc], y)
            del rec, y
        fm, ctx = outs["fnet"], outs["cnet"]
        assert tuple(fm.shape[2:]) == ((h + 7) // 8, (w + 7) // 8)
        fmap1, fmap2 = torch.cat([fm[:-1], fm[1:]]), torch.cat([fm[1:], fm[:-1]])
        cnet = torch.cat([ctx[:-1], ctx[1:]])
        with NL.Recorder({"raft.": model}) as rec:
            low, up = model._refine(fmap1, fmap2, cnet, iters, None, True)
        corr_in = [L.operand for L in rec.launches if getattr(L, "srcs", None) == ["raft.update_block.encoder.convc1"]]
        n, _, h8, w8 = cnet.shape
        coords0 = coords_grid(n, h8, w8).to(DEV)

        def flow(d):
            c = d.glue(lambda t: torch.cat([t[:-1], t[1:]]), ctx)
            return NL.refine(d, "raft.update_block.", c, lambda it, c1: corr_in[it], coords0, iters)
        got_low, got_up = _check(rec, params, f"raft.update[{precision}]", ratios, flow)
        assert len(corr_in) == iters and torch.equal(got_low, low) and torch.equal(got_up, up)
        del rec, outs, fm, ctx, fmap1, fmap2, cnet, corr_in
    _report(f"RAFT [{precision}]", ratios, t0)
