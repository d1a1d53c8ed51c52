"""RAFT correlation / update block and the stage-2 networks through the C ABI against the oracles
(fp32 CUDA-core kernels; tolerance 1e-4 absolute on O(1) outputs, correlation volume 1e-4 relative)."""
import os
import types

import numpy as np
import pytest
import torch

from nets_common import seeded_weights
from oracle import flow_oracle as FO
from oracle import stage2_oracle as SO

pytestmark = pytest.mark.gpu
DEV = "cuda"


def test_corr_build_and_lookup(golden_dir):
    from b200 import nn as K
    from src.models.stage_1.core.corr import CorrBlock
    z = np.load(os.path.join(golden_dir, "raft_corr.npz"))
    f1, f2, coords = (torch.from_numpy(z[k]) for k in ("f1", "f2", "coords"))
    pyr = FO.corr_pyramid(f1, f2)
    blk = CorrBlock(f1.to(DEV), f2.to(DEV), num_levels=4, radius=4)
    flat = torch.cat([p.reshape(-1) for p in pyr])
    got = blk.pyramid.cpu()
    assert got.numel() == flat.numel()
    assert (got - flat).abs().max() <= 1e-4 * flat.abs().max()
    # both builders (wgmma with split fp16 operands = default, fp32 CUDA-core GEMM) to the same fp32-grade bound
    for impl in ("tc", "simt"):
        alt = K.corr_build(f1.to(DEV), f2.to(DEV), impl=impl).cpu()
        err = ((alt - flat).abs().max() / flat.abs().max()).item()
        print(f"corr_build[{impl}] relative error {err:.2e}")
        assert err <= 1e-4
    # a feature map that is not a multiple of the 128-pixel tile, with large and tiny magnitudes
    g = torch.Generator().manual_seed(3)
    a1 = torch.randn(1, 256, 19, 37, generator=g) * torch.logspace(-3, 1.5, 256).view(1, 256, 1, 1)
    a2 = torch.randn(1, 256, 19, 37, generator=g)
    want = torch.cat([p.reshape(-1) for p in FO.corr_pyramid(a1, a2)])
    have = K.corr_build(a1.to(DEV), a2.to(DEV), impl="tc").cpu()
    assert ((have - want).abs().max() / want.abs().max()).item() <= 1e-4
    look = blk(coords.to(DEV)).cpu()
    ref = FO.corr_lookup(pyr, coords)
    assert look.shape == ref.shape == (1, 324, 16, 24)
    assert (look - ref).abs().max() <= 2e-4 * ref.abs().max()
    # out-of-range windows read zeros (grid_sample zeros padding)
    far = coords.clone(); far[:, 0] += 500.0
    assert float(blk(far.to(DEV)).abs().max()) == 0.0


def test_update_block_and_convex_upsample(golden_dir):
    from b200 import nn as K
    from src.models.stage_1.core.update import BasicUpdateBlock
    fx = torch.load(os.path.join(golden_dir, "raft_update.pt"))
    z = np.load(os.path.join(golden_dir, "raft_corr.npz"))
    sd = seeded_weights(fx["shapes"], fx["seed"])
    ub = BasicUpdateBlock(types.SimpleNamespace(corr_levels=4, corr_radius=4), hidden_dim=128)
    ub.load_state_dict(sd)
    ub = ub.to(DEV)
    corr = torch.from_numpy(z["lookup"]).to(DEV)
    net, mask, delta = ub(fx["net"].to(DEV), fx["inp"].to(DEV), corr, fx["flow"].to(DEV))
    o_net, o_mask, o_delta = FO.update_block(sd, fx["net"], fx["inp"], torch.from_numpy(z["lookup"]), fx["flow"])
    assert (net.cpu() - o_net).abs().max() <= 1e-4
    assert (delta.cpu() - o_delta).abs().max() <= 1e-4
    assert (mask.cpu() - o_mask).abs().max() <= 1e-4
    up = K.convex_upsample(fx["flow"].to(DEV), mask)
    assert (up.cpu() - FO.convex_upsample(fx["flow"], o_mask)).abs().max() <= 5e-4


def test_unet_and_transformnet(golden_dir):
    from src.models.network_filter import UNet
    from src.models.network_local import TransformNet
    fx = torch.load(os.path.join(golden_dir, "stage2_nets.pt"))
    unet = UNet(in_channels=6, out_channels=3, init_features=32)
    usd = seeded_weights(fx["unet_shapes"], fx["unet_seed"])
    unet.load_state_dict(usd)
    y = unet.to(DEV)(fx["unet_x"].to(DEV))
    assert (y.cpu() - SO.unet_forward(usd, fx["unet_x"])).abs().max() <= 1e-4
    opts = types.SimpleNamespace(nf=32, norm="IN", model="TransformNet", blocks=5)
    tn = TransformNet(opts, nc_in=12, nc_out=3)
    assert len(tn.state_dict()) == 89
    tsd = seeded_weights(fx["tn_shapes"], fx["tn_seed"])
    tn.load_state_dict(tsd, strict=False)
    yy, (hid, cell) = tn.to(DEV)(fx["tn_x"].to(DEV), None)
    oy, oh, oc = SO.transformnet_forward(tsd, fx["tn_x"])
    assert (yy.cpu() - oy).abs().max() <= 1e-4
    assert (hid.cpu() - oh).abs().max() <= 1e-4
    assert (cell.cpu() - oc).abs().max() <= 1e-4


@pytest.mark.parametrize("mixed", [False, True])
def test_full_raft_against_reference_fixture(golden_dir, mixed):
    """Whole RAFT (encoders with instance / folded batch norm, correlation, 3 update iterations, convex
    upsampling) against outputs of the reference model frozen by make_golden_nets.py (reference on CPU = fp32).
    mixed_precision=False: fp32 CUDA-core convolutions, 2e-3 * max|flow|.  mixed_precision=True: the
    reference's fp16-autocast regime -> wgmma convolutions with fp16 operands, 2e-3 * max|flow| as well
    (measured 1.5e-4; the reference's own autocast execution is not bit-comparable with its fp32 one either)."""
    import argparse
    from src.models.stage_1.core.raft import RAFT
    fx = torch.load(os.path.join(golden_dir, "raft_full.pt"))
    model = RAFT(argparse.Namespace(small=False, mixed_precision=mixed))
    assert len(model.state_dict()) == 179
    model.load_state_dict(seeded_weights(fx["shapes"], fx["seed"]), strict=False)
    model = model.to(DEV).eval()
    low, up = model(fx["im1"].to(DEV), fx["im2"].to(DEV), iters=3, test_mode=True)
    assert low.shape == fx["flow_low"].shape and up.shape == fx["flow_up"].shape == (1, 2, 128, 192)
    tol = 2e-3
    e_low = (low.cpu() - fx["flow_low"]).abs().max().item() / max(fx["flow_low"].abs().max().item(), 1.0)
    e_up = (up.cpu() - fx["flow_up"]).abs().max().item() / max(fx["flow_up"].abs().max().item(), 1.0)
    print(f"RAFT mixed={mixed}: relative error low {e_low:.2e} up {e_up:.2e}")
    assert e_low <= tol and e_up <= tol


# ------------------------------------------------------------------------------------------------
# wgmma convolution (fp16 operands, fp32 accumulation): the operand precision the reference runs these
# layers in (fp16 autocast for RAFT, TF32 cuDNN for stage 2).  Per-layer tolerance 4e-3 * max|y| against an
# fp64 convolution of the same fp32 inputs (operand rounding 2^-11 each, fp32 accumulation); whole-network
# tolerances are stated per test.
CONV_CASES = [
    # n, cin, h, w, cout, kh, kw, stride, pad, pad_mode, act, upsample
    (1, 128, 24, 40, 128, 3, 3, 1, (1, 1), "zeros", "relu", 1),
    (2, 3, 33, 47, 32, 7, 7, 1, (3, 3), "reflect", "leaky", 1),
    (1, 324, 17, 23, 256, 1, 1, 1, (0, 0), "zeros", "relu", 1),
    (1, 384, 16, 24, 128, 1, 5, 1, (0, 2), "zeros", "sigmoid", 1),
    (1, 384, 16, 24, 128, 5, 1, 1, (2, 0), "zeros", "tanh", 1),
    (1, 64, 40, 56, 96, 3, 3, 2, (1, 1), "zeros", "none", 1),
    (1, 64, 20, 28, 32, 3, 3, 1, (1, 1), "reflect", "relu", 2),
    (1, 128, 16, 24, 2, 3, 3, 1, (1, 1), "zeros", "none", 1),
    (1, 256, 16, 24, 576, 1, 1, 1, (0, 0), "zeros", "none", 1),
    (3, 5, 9, 11, 7, 3, 3, 1, (1, 1), "zeros", "none", 1),
    (1, 32, 30, 44, 64, 3, 3, 2, (1, 1), "reflect", "leaky", 1),
    (1, 3, 64, 96, 64, 7, 7, 2, (3, 3), "zeros", "relu", 1),
    (1, 64, 12, 300, 3, 7, 7, 1, (3, 3), "reflect", "tanh", 1),
    (2, 130, 11, 150, 40, 3, 3, 1, (1, 1), "zeros", "none", 2),
]


@pytest.mark.parametrize("case", CONV_CASES)
def test_conv_tc_single_layer(case):
    from b200 import nn as K
    import torch.nn.functional as F
    n, cin, h, w, cout, kh, kw, stride, pad, mode, act, ups = case
    g = torch.Generator().manual_seed(cin * 131 + cout)
    x = torch.randn(n, cin, h, w, generator=g)
    wt = torch.randn(cout, cin, kh, kw, generator=g) / (cin * kh * kw) ** 0.5
    b = torch.randn(cout, generator=g)
    xd, wd, bd = x.to(DEV), wt.to(DEV), b.to(DEV)
    y_tc = K.conv2d(xd, wd, bd, stride=stride, pad=pad, pad_mode=mode, act=act, upsample=ups, precision="tc")
    y_32 = K.conv2d(xd, wd, bd, stride=stride, pad=pad, pad_mode=mode, act=act, upsample=ups, precision="fp32")
    xx = x.double()
    if ups == 2:
        xx = F.interpolate(xx, scale_factor=2, mode="nearest")
    if mode == "reflect":
        xx = F.pad(xx, (pad[1], pad[1], pad[0], pad[0]), mode="reflect")
        ref = F.conv2d(xx, wt.double(), b.double(), stride=stride)
    else:
        ref = F.conv2d(xx, wt.double(), b.double(), stride=stride, padding=pad)
    ref = {"none": lambda t: t, "relu": torch.relu, "leaky": lambda t: F.leaky_relu(t, 0.2),
           "sigmoid": torch.sigmoid, "tanh": torch.tanh}[act](ref)
    assert y_tc.shape == ref.shape == y_32.shape
    scale = ref.abs().max().item()
    assert (y_32.cpu().double() - ref).abs().max() <= 2e-5 * scale
    assert (y_tc.cpu().double() - ref).abs().max() <= 4e-3 * scale        # TMA-fed kernel


def test_conv_tc_slices_residual_and_scale():
    from b200 import _native as N
    from b200 import nn as K
    g = torch.Generator().manual_seed(5)
    x = torch.randn(1, 96, 20, 28, generator=g).to(DEV)
    wt = (torch.randn(40, 64, 3, 3, generator=g) / 24).to(DEV)
    b = torch.randn(40, generator=g).to(DEV)
    res = torch.randn(1, 50, 20, 28, generator=g).to(DEV)
    outs = []
    for prec in ("fp32", "tc"):
        out = torch.full((1, 64, 20, 28), 7.0, device=DEV)
        K.conv2d(x, wt, b, pad=1, act="tanh", out=out, out_c_off=8, in_slice=(16, 80), residual=res, res_c_off=10,
                 out_scale=0.25, precision=prec)
        outs.append(out)
    assert torch.equal(outs[1][:, :8], torch.full_like(outs[1][:, :8], 7.0))
    assert torch.equal(outs[1][:, 48:], torch.full_like(outs[1][:, 48:], 7.0))
    assert (outs[0] - outs[1]).abs().max() <= 4e-3 * outs[0][:, 8:48].abs().max()
    with pytest.raises(N.B200Error, match="stride 1 and 2"):     # no silent fall-back to another arithmetic
        K.conv2d(x, wt, b, stride=3, pad=1, in_slice=(16, 80), precision="tc")


def test_networks_with_tc_convolutions(golden_dir):
    """Update block, UNet and TransformNet with every convolution on wgmma: 2e-2 * max|oracle output|
    (several dozen fp16-operand layers deep; the reference's own fp16/TF32 execution differs from an fp32
    oracle by the same order)."""
    from b200 import nn as K
    from src.models.network_filter import UNet
    from src.models.network_local import TransformNet
    from src.models.stage_1.core.update import BasicUpdateBlock
    prev = K.set_conv_precision("tc")
    try:
        fx = torch.load(os.path.join(golden_dir, "raft_update.pt"))
        z = np.load(os.path.join(golden_dir, "raft_corr.npz"))
        sd = seeded_weights(fx["shapes"], fx["seed"])
        ub = BasicUpdateBlock(types.SimpleNamespace(corr_levels=4, corr_radius=4), hidden_dim=128)
        ub.load_state_dict(sd)
        ub = ub.to(DEV)
        net, mask, delta = ub(fx["net"].to(DEV), fx["inp"].to(DEV), torch.from_numpy(z["lookup"]).to(DEV),
                              fx["flow"].to(DEV))
        o_net, o_mask, o_delta = FO.update_block(sd, fx["net"], fx["inp"], torch.from_numpy(z["lookup"]), fx["flow"])
        errs = {"net": ((net.cpu() - o_net).abs().max() / o_net.abs().max()).item(),
                "delta": ((delta.cpu() - o_delta).abs().max() / o_delta.abs().max()).item(),
                "mask": ((mask.cpu() - o_mask).abs().max() / o_mask.abs().max()).item()}
        fx = torch.load(os.path.join(golden_dir, "stage2_nets.pt"))
        unet = UNet(in_channels=6, out_channels=3, init_features=32)
        usd = seeded_weights(fx["unet_shapes"], fx["unet_seed"])
        unet.load_state_dict(usd)
        y = unet.to(DEV)(fx["unet_x"].to(DEV))
        oy = SO.unet_forward(usd, fx["unet_x"])
        errs["unet"] = ((y.cpu() - oy).abs().max() / oy.abs().max()).item()
        tn = TransformNet(types.SimpleNamespace(nf=32, norm="IN", model="TransformNet", blocks=5), nc_in=12, nc_out=3)
        tsd = seeded_weights(fx["tn_shapes"], fx["tn_seed"])
        tn.load_state_dict(tsd, strict=False)
        yy, (hid, cell) = tn.to(DEV)(fx["tn_x"].to(DEV), None)
        oy, oh, oc = SO.transformnet_forward(tsd, fx["tn_x"])
        errs["tn"] = ((yy.cpu() - oy).abs().max() / oy.abs().max()).item()
        errs["tn_cell"] = ((cell.cpu() - oc).abs().max() / oc.abs().max()).item()
        print("tc network errors (relative to max):", errs)
        assert max(errs.values()) <= 2e-2, errs
    finally:
        K.set_conv_precision(prev)


def test_conv_tc_fused_bilinear_upsample():
    """nn.Upsample(scale_factor=2, mode='bilinear', align_corners=True) + Conv2d (UNet upconv, network_filter.py:22):
    fused into the fp16 repack on the wgmma path, explicit kernel + fp32 convolution otherwise."""
    from b200 import nn as K
    import torch.nn.functional as F
    g = torch.Generator().manual_seed(11)
    x = torch.randn(1, 70, 17, 29, generator=g)
    wt = torch.randn(40, 70, 3, 3, generator=g) / 25.0
    b = torch.randn(40, generator=g)
    ref = F.conv2d(F.interpolate(x.double(), scale_factor=2, mode="bilinear", align_corners=True), wt.double(), b.double(),
                   padding=1)
    scale = ref.abs().max().item()
    y32 = K.conv2d(x.to(DEV), wt.to(DEV), b.to(DEV), pad=1, upsample=2, upsample_mode="bilinear", precision="fp32")
    ytc = K.conv2d(x.to(DEV), wt.to(DEV), b.to(DEV), pad=1, upsample=2, upsample_mode="bilinear", precision="tc")
    assert y32.shape == ytc.shape == ref.shape
    assert (y32.cpu().double() - ref).abs().max() <= 2e-5 * scale
    assert (ytc.cpu().double() - ref).abs().max() <= 4e-3 * scale


def test_raft_both_directions_share_the_encoder(golden_dir):
    """forward_both (one fnet pass) == two independent forward calls, bit for bit."""
    import argparse
    from src.models.stage_1.core.raft import RAFT
    fx = torch.load(os.path.join(golden_dir, "raft_full.pt"))
    model = RAFT(argparse.Namespace(small=False, mixed_precision=True))
    model.load_state_dict(seeded_weights(fx["shapes"], fx["seed"]), strict=False)
    model = model.to(DEV).eval()
    a, b = fx["im1"].to(DEV), fx["im2"].to(DEV)
    (lo12, up12), (lo21, up21) = model.forward_both(a, b, iters=3)
    r12 = model(a, b, iters=3, test_mode=True)
    r21 = model(b, a, iters=3, test_mode=True)
    assert torch.equal(up12, r12[1]) and torch.equal(lo12, r12[0])
    assert torch.equal(up21, r21[1]) and torch.equal(lo21, r21[0])


def test_chained_convolutions_equal_unchained():
    """conv -> conv with the intermediate written by the first epilogue straight into the second one's packed fp16 input
    (b200_conv2d_tma_chain) against the same two wgmma convolutions with an fp32 tensor + repack in between: the
    consumer sees the same fp16 operands, so the results are bit-identical.  Also a two-producer concat (192 + 64
    channels, RAFT motion encoder) and an odd width (ragged last tile)."""
    from b200 import nn as K
    g = torch.Generator().manual_seed(31)
    prev = K.set_conv_precision("tc")
    try:
        for (n, cin, h, w, mid, cout) in ((1, 6, 24, 37, 32, 32), (1, 64, 19, 130, 96, 40), (2, 32, 16, 24, 128, 8)):
            x = torch.randn(n, cin, h, w, generator=g).to(DEV)
            w1 = (torch.randn(mid, cin, 3, 3, generator=g) / (3 * cin ** 0.5)).to(DEV)
            w2 = (torch.randn(cout, mid, 3, 3, generator=g) / (3 * mid ** 0.5)).to(DEV)
            b2 = torch.randn(cout, generator=g).to(DEV)
            t = K.conv2d(x, w1, None, pad=1, act="relu")
            ref = K.conv2d(t, w2, b2, pad=1, act="tanh")
            ch = K.Chain(n, mid, h, w, (3, 3), 1, DEV)
            both = K.conv2d(x, w1, None, pad=1, act="relu", chain_out=ch)           # fp32 AND packed
            assert torch.equal(both, t)
            got = K.conv2d(ch, w2, b2, pad=1, act="tanh")
            assert torch.equal(got, ref), float((got - ref).abs().max())
            assert K.conv2d(x, w1, None, pad=1, act="relu", chain_out=ch, keep_fp32=False) is None
            assert torch.equal(K.conv2d(ch, w2, b2, pad=1, act="tanh"), ref)
        # two producers fill one consumer input (torch.cat in the reference, core/update.py:95)
        a = torch.randn(1, 256, 17, 29, generator=g).to(DEV); bsrc = torch.randn(1, 128, 17, 29, generator=g).to(DEV)
        wa = (torch.randn(192, 256, 3, 3, generator=g) / 48).to(DEV); wb = (torch.randn(64, 128, 3, 3, generator=g) / 34).to(DEV)
        wc = (torch.randn(126, 256, 3, 3, generator=g) / 48).to(DEV)
        cat = torch.empty(1, 256, 17, 29, device=DEV)
        K.conv2d(a, wa, None, pad=1, act="relu", out=cat, out_c_off=0)
        K.conv2d(bsrc, wb, None, pad=1, act="relu", out=cat, out_c_off=192)
        ref = K.conv2d(cat, wc, None, pad=1, act="relu")
        ch = K.Chain(1, 256, 17, 29, (3, 3), 1, DEV, tag="test_concat")
        K.conv2d(a, wa, None, pad=1, act="relu", chain_out=ch, chain_c_off=0, keep_fp32=False)
        K.conv2d(bsrc, wb, None, pad=1, act="relu", chain_out=ch, chain_c_off=192, keep_fp32=False)
        assert torch.equal(K.conv2d(ch, wc, None, pad=1, act="relu"), ref)
        with pytest.raises(Exception):
            K.Chain(1, 8, 16, 16, (3, 3), 1, DEV)          # 8 channels x 3 taps are folded: not chainable
    finally:
        K.set_conv_precision(prev)


def test_chained_reflection_padded_convolution():
    """A chained consumer with nn.ReflectionPad2d: the consumer call mirrors the interior of the packed buffer into its
    halo before the convolution (7x7 / pad 3 and 3x3 / pad 1): bit-identical with the unchained wgmma pair."""
    from b200 import nn as K
    g = torch.Generator().manual_seed(32)
    prev = K.set_conv_precision("tc")
    try:
        for (cin, mid, cout, k, h, w) in ((16, 64, 3, 7, 21, 45), (32, 128, 128, 3, 18, 34)):
            x = torch.randn(1, cin, h, w, generator=g).to(DEV)
            w1 = (torch.randn(mid, cin, 3, 3, generator=g) / (3 * cin ** 0.5)).to(DEV)
            w2 = (torch.randn(cout, mid, k, k, generator=g) / (k * mid ** 0.5)).to(DEV)
            t = K.conv2d(x, w1, None, pad=1, pad_mode="reflect", act="leaky")
            ref = K.conv2d(t, w2, None, pad=k // 2, pad_mode="reflect", act="tanh")
            ch = K.Chain(1, mid, h, w, (k, k), k // 2, DEV, pad_mode="reflect", tag="test_reflect")
            K.conv2d(x, w1, None, pad=1, pad_mode="reflect", act="leaky", chain_out=ch, keep_fp32=False)
            got = K.conv2d(ch, w2, None, pad=k // 2, pad_mode="reflect", act="tanh")
            assert torch.equal(got, ref), float((got - ref).abs().max())
    finally:
        K.set_conv_precision(prev)
