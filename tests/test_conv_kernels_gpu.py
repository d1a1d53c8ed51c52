"""Kernel-level tests of the convolutions: the tensor-core path of csrc/conv_tma.cu (repack, TMA/wgmma kernel, reflection
halo, weight images, chained fp16 outputs) and the fp32 `conv2d_kernel` of csrc/conv_simt.cu, one layer at a time,
against the operand-exact float64 reference of conv_common.py (its bound is stated there).

The constants were set from one run on an H100 80GB HBM3 at a 400 W power limit, at about 10x the largest measured
ratio (printed by `pytest -s` next to every case).  The largest ratios, 0.45 on the wgmma path and 0.49 on the CUDA-core
path, both come from the 9-tap case `fold_cin1`, so C_TC = C_FP32 = 4.  For long reductions the wgmma path's ratio
is the larger one (0.12-0.16 at R = 3456 and 12384, against 0.02-0.08), but it does not grow with R.  The error thus
grows no faster than sqrt(R), and the bound keeps sqrt(R) on both paths: no truncating accumulation inside the MMA
shows up at these lengths.

Every case runs on both paths.  It names the branch of the tensor-core planner (`tma_geometry` / `launch_conv_tma`) it
exists for, and a Python mirror of that planner, kept here, asserts that the case lands in it; a CPU test checks that
the table covers every branch and that the mirror agrees with the library's image and workspace sizes.  Besides the
bound, every case checks that the output slice is finite and that the channels outside it keep a sentinel value."""
import ctypes as C
import math
import zlib

import pytest
import torch
import torch.nn.functional as F

from b200 import _native as N
from b200 import nn as K
from conv_common import ACTS, C_FP32, C_TC, bound_ratio, chain_view, reference
from csrc_build import ensure_built

DEV = "cuda"
SENTINEL = -12345.0
H100_SMS = 132


# ---------------------------------------------------------------------------------------------------------------
# Mirror of the tensor-core planner (csrc/conv_tma.cu: tma_geometry, launch_conv_tma), split operands excluded
# ---------------------------------------------------------------------------------------------------------------
def _cdiv(a, b):
    return -(-a // b)


def plan(c):
    kh, kw = c["k"]
    ph, pw = c["pad"]
    s, up = c["stride"], c["upsample"]
    hp, wp = c["h"] * up + 2 * ph, c["w"] * up + 2 * pw
    oh, ow = (hp - kh) // s + 1, (wp - kw) // s + 1
    phases, shift = (4, 1) if s == 2 else (1, 0)
    hp2, wp2 = _cdiv(hp, s), _cdiv(wp, s)
    cchunks = _cdiv(c["cin"], 64)
    n_chunks = kh * kw * cchunks
    cf = _cdiv(c["cin"], 8) * 8
    fold_cf = cf if s == 1 and kw > 1 and cf * kw <= 64 and c["up_mode"] == "nearest" else 0
    if fold_cf:
        wp2, n_chunks = ow, kh
    kw_eff = 1 if fold_cf else kw
    n_tiles_n = _cdiv(c["cout"], 256)
    per_tile = _cdiv(c["cout"], n_tiles_n)
    n_tile = 64 if per_tile <= 64 else 128 if per_tile <= 128 else 256
    b_bytes = n_tile * 128
    nsub = _cdiv(kw_eff, s)
    resident = n_tiles_n == 1 and n_chunks * b_bytes <= 100 * 1024
    b_group = 1 if resident else max(1, min(32768 // b_bytes, nsub))
    x_tiles = _cdiv(ow, 128)
    return dict(oh=oh, ow=ow, fold_cf=fold_cf, n_tile=n_tile, n_tiles_n=n_tiles_n, resident=resident, b_group=b_group,
                nsub=nsub, phases=phases, a_rows=128 + ((kw_eff - 1) >> shift), x_tiles=x_tiles, n_chunks=n_chunks,
                total_tiles=c["n"] * oh * x_tiles * n_tiles_n,
                image_bytes=n_tiles_n * n_chunks * n_tile * 128,
                workspace_bytes=c["n"] * phases * hp2 * wp2 * cchunks * 64 * 2 + 256)


# ---------------------------------------------------------------------------------------------------------------
# Case table: each case names the planner branch it exists for and the planner fields it must land on
# ---------------------------------------------------------------------------------------------------------------
CASES = {}


def spec(name, branch="", expect=None, n=1, cin=40, h=6, w=20, cout=32, k=(3, 3), stride=1, pad=(1, 1), pad_mode="zeros",
         act="none", upsample=1, up_mode="nearest", in_slice=None, out_slice=None, res_slice=None, bias=True,
         out_scale=1.0, saturate=False):
    """One convolution: in_slice = (first channel, channels of x), out_slice / res_slice likewise for the output and
    the residual tensor."""
    return dict(name=name, branch=branch, expect=expect or {}, n=n, cin=cin, h=h, w=w, cout=cout, k=k, stride=stride,
                pad=pad, pad_mode=pad_mode, act=act, upsample=upsample, up_mode=up_mode, in_slice=in_slice,
                out_slice=out_slice, res_slice=res_slice, bias=bias, out_scale=out_scale, saturate=saturate)


def _case(name, branch, expect, **kw):
    CASES[name] = spec(name, branch, expect, **kw)


COUTS = (1, 2, 8, 63, 64, 65, 128, 129, 192, 256, 257, 300, 576)
for _co in COUTS:
    _tiles = _cdiv(_co, 256)
    _per = _cdiv(_co, _tiles)
    _case(f"cout{_co}", "N tile width and count; padded weight rows in the last tile",
          dict(n_tile=64 if _per <= 64 else 128 if _per <= 128 else 256, n_tiles_n=_tiles, fold_cf=0), cout=_co)

# resident weight image (n_tiles_n == 1 and <= 100 KB) against streamed weights, on both sides of the line
_case("resident_n64_12chunks", "resident: 12 chunks of n_tile 64 = 96 KB", dict(n_tile=64, n_chunks=12, resident=True),
      k=(3, 4), pad=(1, 2), cout=64, w=21)
_case("streamed_n64_13chunks", "streamed: 13 chunks of n_tile 64 = 104 KB", dict(n_tile=64, n_chunks=13, resident=False),
      k=(13, 1), pad=(6, 0), h=15, cout=64)
_case("resident_n256_cin192", "resident: 3 chunks of n_tile 256", dict(n_tile=256, n_chunks=3, resident=True),
      cin=192, k=(1, 1), pad=(0, 0), cout=256, h=5, w=30)
_case("streamed_n256_cin193", "streamed: 4 chunks of n_tile 256, one-channel k-step tail",
      dict(n_tile=256, n_chunks=4, resident=False), cin=193, k=(1, 1), pad=(0, 0), cout=256, h=5, w=30)
# x taps per weight stage with a ragged last stage
_case("bgroup_4_3", "streamed, 7 x taps in stages of 4 and 3", dict(n_tile=64, b_group=4, nsub=7, resident=False, fold_cf=0),
      cin=96, k=(1, 7), pad=(0, 3), cout=64, h=4, w=40)
_case("bgroup_2_2_1", "streamed, 5 x taps in stages of 2, 2 and 1", dict(n_tile=128, b_group=2, nsub=5, resident=False),
      cin=96, k=(1, 5), pad=(0, 2), cout=128, h=4, w=40)
_case("bgroup_n256", "streamed n_tile 256: one tap per stage", dict(n_tile=256, b_group=1, nsub=3, resident=False),
      cin=64, k=(3, 3), cout=200, h=5, w=30)
# both rings wrap their phase many times per CTA
for _co in (64, 128, 256):
    _case(f"ring_wrap_n{_co}", "tiles several times the SM count, 54 chunks per tile",
          dict(n_tile=_co, resident=False, n_chunks=54), n=5, cin=384, h=100, w=5, cout=_co)
# x taps folded into the channel vector, both sides of cf * KW <= 64
_case("fold_cin8_kw7", "folded: 8 x 7 = 56 slots", dict(fold_cf=8, n_chunks=7, a_rows=128), cin=8, k=(7, 7), pad=(3, 3),
      h=12, w=40)
_case("nofold_cin9_kw7", "not folded: 16 x 7 = 112 slots", dict(fold_cf=0, a_rows=134), cin=9, k=(7, 7), pad=(3, 3),
      h=12, w=40)
_case("fold_cin32_kw2", "folded: exactly 64 slots", dict(fold_cf=32, n_chunks=2), cin=32, k=(2, 2), pad=(0, 0), h=9, w=33)
_case("fold_cin16_kw3", "folded: 48 slots", dict(fold_cf=16, n_chunks=3), cin=16, k=(3, 3), h=9, w=33)
_case("nofold_cin21_kw3", "not folded: 72 slots", dict(fold_cf=0, n_chunks=9), cin=21, k=(3, 3), h=9, w=33)
_case("fold_cin1", "folded: one input channel", dict(fold_cf=8), cin=1, k=(3, 3), h=11, w=29)
_case("fold_reflect", "folded with reflection padding", dict(fold_cf=8), cin=6, k=(7, 7), pad=(3, 3), pad_mode="reflect",
      h=13, w=37, act="leaky")
_case("fold_nearest2", "folded with nearest x2", dict(fold_cf=8), cin=5, k=(3, 3), upsample=2, h=7, w=19)
_case("fold_batch3", "folded with N > 1", dict(fold_cf=8), n=3, cin=3, k=(5, 5), pad=(2, 2), h=9, w=21)
_case("fold_in_slice_3", "folded, input channel slice at an odd offset", dict(fold_cf=8), cin=4, in_slice=(3, 11),
      k=(3, 3), h=9, w=21)
# stride 2: the 4 pixel phases; odd H and W give phase planes of different extents; stride 2 never folds
for _kh in (1, 3):
    for _kw in (1, 3, 4, 7):
        _case(f"s2_{_kh}x{_kw}", "stride 2: phase split", dict(phases=4, fold_cf=0, a_rows=128 + ((_kw - 1) >> 1)),
              stride=2, cin=(64 if (_kh, _kw) == (1, 1) else 4 if _kw == 3 else 24), k=(_kh, _kw), pad=(_kh // 2, _kw // 2),
              h=13, w=21)
_case("s2_reflect", "stride 2 with reflection padding", dict(phases=4), stride=2, cin=32, pad_mode="reflect", h=15,
      w=23, act="leaky")
_case("s2_nearest2", "stride 2 of a nearest x2 input", dict(phases=4, fold_cf=0), stride=2, upsample=2, cin=12, h=7, w=11)
# A box wider than 128 pixel rows
_case("abox_1x15", "a_rows 142", dict(a_rows=142, fold_cf=0), cin=96, k=(1, 15), pad=(0, 7), h=2, w=300)
_case("abox_1x31", "a_rows 158", dict(a_rows=158, fold_cf=0), cin=96, k=(1, 31), pad=(0, 15), h=2, w=300)
_case("abox_1x129", "a_rows 256, the widest box", dict(a_rows=256, fold_cf=0), cin=96, k=(1, 129), pad=(0, 64), h=1,
      w=150)
# ragged pixel tiles; with N = 3 and OH = 1 the 128-pixel tiles follow each other across images
for _ow in (1, 127, 128, 129, 255, 257):
    _case(f"ow{_ow}", "ragged last pixel tile", dict(x_tiles=_cdiv(_ow, 128), fold_cf=0), n=3, cin=24, h=1, w=_ow, cout=40)
# repack
_case("pack_wp2_47", "packed width 47: not a multiple of the 32-pixel block, two channel blocks with a tail",
      dict(fold_cf=0), cin=70, h=5, w=45)
_case("pack_in_slice_3", "input channels 3..43 of 80, k-step tail", dict(fold_cf=0), cin=40, in_slice=(3, 80), h=7, w=23)
_case("pack_in_slice_61", "input channels 61..161 of 200, second channel block 36 wide", dict(fold_cf=0), cin=100,
      in_slice=(61, 200), h=7, w=23)
_case("bilinear_h1", "bilinear x2 from one row", dict(fold_cf=0), cin=20, upsample=2, up_mode="bilinear", h=1, w=9)
_case("bilinear_w1", "bilinear x2 from one column", dict(fold_cf=0), cin=20, upsample=2, up_mode="bilinear", h=9, w=1)
_case("bilinear_reflect", "bilinear x2 with reflection padding", dict(fold_cf=0), cin=3, upsample=2, up_mode="bilinear",
      pad_mode="reflect", h=8, w=13)
_case("bilinear_stride2", "bilinear x2 with stride 2", dict(phases=4), cin=20, upsample=2, up_mode="bilinear", stride=2,
      h=7, w=10)
_case("reflect_pad_size_minus_1", "reflection pads H - 1 and W - 1", dict(fold_cf=0), cin=16, k=(7, 9), pad=(3, 4),
      pad_mode="reflect", h=4, w=5)
# epilogue
for _a in ("relu", "leaky", "sigmoid", "tanh"):
    _case(f"act_{_a}", "epilogue activation", dict(), act=_a, cin=48, cout=72, h=7, w=30)
_case("out_scale", "epilogue scale", dict(), act="tanh", out_scale=0.37)
_case("residual_offset", "residual channels 5..45 of 50 after the scale", dict(), cout=40, act="relu", out_scale=0.5,
      res_slice=(5, 50))
_case("no_bias", "epilogue without bias", dict(), bias=False, cout=48)
_case("out_slice", "output channels 7..39 of 60, sentinel elsewhere", dict(), out_slice=(7, 60))
# fp16 saturation of both operands
_case("saturate", "operands beyond +-65504 saturate in the repack and the weight images", dict(fold_cf=0), cin=24,
      cout=40, saturate=True)


def _inputs(c):
    g = torch.Generator().manual_seed(zlib.crc32(c["name"].encode()))
    c_total = c["cin"] if c["in_slice"] is None else c["in_slice"][1]
    kh, kw = c["k"]
    x = torch.randn(c["n"], c_total, c["h"], c["w"], generator=g)
    w = torch.randn(c["cout"], c["cin"], kh, kw, generator=g) / math.sqrt(c["cin"] * kh * kw)
    b = torch.randn(c["cout"], generator=g) if c["bias"] else None
    if c["saturate"]:                                       # some operands beyond the fp16 range, both signs
        x.view(-1)[::7] *= 9e4
        x.view(-1)[3::11] = 65519.0                         # rounds to 65504 (RN) ...
        x.view(-1)[5::13] = -65520.0                        # ... and to -inf without saturation
        w.view(-1)[::5] = 7e4 * w.view(-1)[::5].sign()
        w.view(-1)[2::17] = -1e6
    p = plan(c)
    res = None
    if c["res_slice"] is not None:
        res = torch.randn(c["n"], c["res_slice"][1], p["oh"], p["ow"], generator=g)
    return x, w, b, res


def run_case(c, x, w, b, res, precision, weight=None):
    """Run one case on the device into a sentinel-filled output; returns the whole output tensor on the CPU."""
    p = plan(c)
    o_off, o_total = c["out_slice"] or (0, c["cout"])
    out = torch.full((c["n"], o_total, p["oh"], p["ow"]), SENTINEL, device=DEV)
    K.conv2d(x.to(DEV), weight if weight is not None else w.to(DEV), None if b is None else b.to(DEV),
             stride=c["stride"], pad=c["pad"], pad_mode=c["pad_mode"], act=c["act"], upsample=c["upsample"],
             upsample_mode=c["up_mode"], out=out, out_c_off=o_off,
             in_slice=None if c["in_slice"] is None else (c["in_slice"][0], c["in_slice"][0] + c["cin"]),
             residual=None if res is None else res.to(DEV), res_c_off=0 if res is None else c["res_slice"][0],
             out_scale=c["out_scale"], precision=precision)
    return out.cpu()


def check_layer(c, out, y_ref, slack, unit, tc, what):
    """Sentinel outside the output slice, finite inside, and the elementwise bound; prints the measured constant."""
    o_off, o_total = c["out_slice"] or (0, c["cout"])
    assert torch.equal(out[:, :o_off], torch.full_like(out[:, :o_off], SENTINEL)), what
    assert torch.equal(out[:, o_off + c["cout"]:], torch.full_like(out[:, o_off + c["cout"]:], SENTINEL)), what
    y = out[:, o_off:o_off + c["cout"]].double()
    assert torch.isfinite(y).all(), f"{what}: non-finite output"
    const = C_TC if tc else C_FP32
    ratio, bad, err_max = bound_ratio(y, y_ref, slack, unit, const)
    kh, kw = c["k"]
    r = c["cin"] * kh * kw
    print(f"{what}: err/(u*sqrt(R)*A) = {ratio:.3f}  [linear in R: {ratio / math.sqrt(r):.4f}]  bound c = {const:g}"
          f"  max err {err_max:.3e}")
    assert not bad, f"{what}: {bad} elements beyond the bound, ratio {ratio:.3f} > {const:g}"


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["tc", "fp32"])
@pytest.mark.parametrize("name", list(CASES))
def test_conv_layer(name, precision):
    """One convolution against the operand-exact float64 reference (bound in the module docstring)."""
    c = CASES[name]
    p = plan(c)
    for key, val in c["expect"].items():
        assert p[key] == val, (name, key, p[key], val)
    x, w, b, res = _inputs(c)
    out = run_case(c, x, w, b, res, precision)
    tc = precision == "tc"
    check_layer(c, out, *reference(c, x, w, b, res, tc), tc, f"{name}[{precision}]")


# ---------------------------------------------------------------------------------------------------------------
# Chained convolutions: the producer's epilogue writes fp16 straight into the consumer's packed input
# ---------------------------------------------------------------------------------------------------------------
def _randn(g, *shape, scale=1.0):
    return torch.randn(*shape, generator=g) * scale


def _chain_view(ch, c):
    return chain_view(ch, c["n"], c["cin"], c["h"], c["w"], c["pad"])


@pytest.mark.gpu
@pytest.mark.parametrize("c_off", [0, 8])
def test_chained_consumer_against_reference(c_off):
    """A producer writes 16 channels at offset c_off of a 36-channel packed input (zero padding) whose other channels,
    and the channel padding up to 64, hold earlier values.  After the producer: the slice holds
    fp16(satfinite(producer fp32 output)) of the same call, every other element is unchanged and the halo is still
    zero.  The consumer (3 k16 steps, the last one half padding) is then checked against the reference on exactly
    that input."""
    g = torch.Generator().manual_seed(40 + c_off)
    n, h, w = 2, 10, 37
    cons = spec("chain_consumer", n=n, cin=36, h=h, w=w, cout=40, act="tanh")
    x, w1, b1 = _randn(g, n, 24, h, w), _randn(g, 16, 24, 3, 3, scale=216 ** -0.5), _randn(g, 16)
    w2, b2 = _randn(g, 40, 36, 3, 3, scale=324 ** -0.5), _randn(g, 40)
    ch = K.Chain(n, 36, h, w, (3, 3), 1, DEV, tag=f"test_conv_kernels_{c_off}")
    view = _chain_view(ch, cons)
    view.zero_()
    view[:, 1:1 + h, 1:1 + w, :] = _randn(g, n, h, w, view.shape[3]).half().to(DEV)
    before = view.clone()
    y = K.conv2d(x.to(DEV), w1.to(DEV), b1.to(DEV), pad=1, act="leaky", chain_out=ch, chain_c_off=c_off)
    want = before.clone()
    want[:, 1:1 + h, 1:1 + w, c_off:c_off + 16] = y.permute(0, 2, 3, 1).clamp(-65504, 65504).half()
    assert torch.equal(view, want)
    halo = torch.ones_like(view, dtype=torch.bool)
    halo[:, 1:1 + h, 1:1 + w] = False
    assert not bool(view[halo].any()), "the zero halo was written"
    z = K.conv2d(ch, w2.to(DEV), b2.to(DEV), pad=1, act="tanh")
    t = want[:, 1:1 + h, 1:1 + w, :36].permute(0, 3, 1, 2).float().cpu()
    check_layer(cons, z.cpu(), *reference(cons, t, w2, b2, None, True), True, f"chained consumer c_off {c_off}")


@pytest.mark.gpu
@pytest.mark.parametrize("k,pad", [((1, 7), (0, 3)), ((7, 1), (3, 0)), ((3, 7), (1, 3))])
def test_chained_reflection_halo(k, pad):
    """Reflection padding of a chained input with asymmetric pads, reaching every branch of conv_reflect_halo_kernel
    (no top / bottom band, no side columns, both): the consumer against the reference, and the halo of the packed
    buffer equal to the reflection of its interior in every channel."""
    g = torch.Generator().manual_seed(50 + k[0] * 8 + k[1])
    n, h, w = 1, 9, 13
    cons = spec("chain_reflect", n=n, cin=16, h=h, w=w, cout=24, k=k, pad=pad, pad_mode="reflect")
    x, w1 = _randn(g, n, 8, h, w), _randn(g, 16, 8, 3, 3, scale=72 ** -0.5)
    w2, b2 = _randn(g, 24, 16, *k, scale=(16 * k[0] * k[1]) ** -0.5), _randn(g, 24)
    ch = K.Chain(n, 16, h, w, k, pad, DEV, tag="test_conv_kernels_reflect", pad_mode="reflect")
    y = K.conv2d(x.to(DEV), w1.to(DEV), None, pad=1, pad_mode="reflect", act="relu", chain_out=ch)
    z = K.conv2d(ch, w2.to(DEV), b2.to(DEV), pad=pad, pad_mode="reflect")
    check_layer(cons, z.cpu(), *reference(cons, y.cpu(), w2, b2, None, True), True, f"chained reflect {k} pad {pad}")
    view = _chain_view(ch, cons).cpu()
    ph, pw = pad
    inner = view[:, ph:ph + h, pw:pw + w].permute(0, 3, 1, 2).float()
    assert torch.equal(view, F.pad(inner, (pw, pw, ph, ph), mode="reflect").permute(0, 2, 3, 1).half())


@pytest.mark.gpu
def test_chained_overflow_saturates_like_the_repack():
    """Producer outputs beyond +-65504: the chained fp16 store saturates as the repack of an unchained consumer does,
    so both consumers are finite and bit-identical."""
    g = torch.Generator().manual_seed(60)
    x, w1 = _randn(g, 1, 8, 6, 20).to(DEV), _randn(g, 24, 8, 3, 3, scale=3e4 / 72 ** 0.5).to(DEV)
    w2, b2 = _randn(g, 16, 24, 3, 3, scale=1e-4).to(DEV), _randn(g, 16).to(DEV)
    t = K.conv2d(x, w1, None, pad=1, precision="tc")
    assert float(t.abs().max()) > 65504.0
    ref = K.conv2d(t, w2, b2, pad=1, precision="tc")
    ch = K.Chain(1, 24, 6, 20, (3, 3), 1, DEV, tag="test_conv_kernels_overflow")
    assert K.conv2d(x, w1, None, pad=1, chain_out=ch, keep_fp32=False) is None
    got = K.conv2d(ch, w2, b2, pad=1)
    assert bool(torch.isfinite(got).all()) and bool(torch.isfinite(ref).all())
    assert torch.equal(got, ref), float((got - ref).abs().max())


# ---------------------------------------------------------------------------------------------------------------
# Weight-image cache
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_weight_image_cache_follows_the_fold_decision():
    """One narrow weight (3 -> 8 channels, 3x3) used with bilinear x2 (x taps not folded: 9 chunks) and then with
    nearest x2 (folded: 3 chunks).  The image depends on that decision, so the second call must not reuse the first
    one's image."""
    g = torch.Generator().manual_seed(70)
    x, w, b = _randn(g, 1, 3, 7, 9), _randn(g, 8, 3, 3, 3, scale=27 ** -0.5), _randn(g, 8)
    wd = w.to(DEV)
    for mode, fold in (("bilinear", 0), ("nearest", 8)):
        c = spec(f"cache_{mode}", cin=3, h=7, w=9, cout=8, upsample=2, up_mode=mode)
        assert plan(c)["fold_cf"] == fold
        out = run_case(c, x, w, b, None, "tc", weight=wd)
        check_layer(c, out, *reference(c, x, w, b, None, True), True, f"cached weight, {mode}")


@pytest.mark.gpu
def test_weight_image_cache_follows_rebinding():
    """`w.data = other` keeps the tensor object and its version: the next call must use the new values."""
    c = spec("cache_rebind", cout=64)
    x, w, b, _ = _inputs(c)
    wd = w.to(DEV)
    run_case(c, x, w, b, None, "tc", weight=wd)
    w_new = torch.flip(w, dims=(0,)) * 0.5
    wd.data = w_new.to(DEV)
    out = run_case(c, x, w_new, b, None, "tc", weight=wd)
    check_layer(c, out, *reference(c, x, w_new, b, None, True), True, "cached weight after w.data = other")


# ---------------------------------------------------------------------------------------------------------------
# Planner coverage and host-side refusals (no GPU needed)
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    ensure_built()
    return N.lib()


def _desc(c):
    lo, total = (0, c["cin"]) if c["in_slice"] is None else (c["in_slice"][0], c["in_slice"][1])
    o_off, o_total = c["out_slice"] or (0, c["cout"])
    r_off, r_total = c["res_slice"] or (0, 0)
    return N.ConvDesc(c["n"], c["cin"], c["h"], c["w"], total, lo, c["cout"], c["k"][0], c["k"][1], c["stride"],
                      c["pad"][0], c["pad"][1], 1 if c["pad_mode"] == "reflect" else 0, c["upsample"], o_total, o_off,
                      K.ACT[c["act"]], c["out_scale"], r_total, r_off, 1 if c["up_mode"] == "bilinear" else 0)


def test_case_table_covers_the_planner(lib):
    """Every case lands in the branch it names, the planner mirror agrees with the library's weight-image and
    workspace sizes, and the table reaches every branch of the planner, repack and epilogue."""
    plans = {}
    for name, c in CASES.items():
        p = plans[name] = plan(c)
        for key, val in c["expect"].items():
            assert p[key] == val, (name, key, p[key], val)
        d = _desc(c)
        assert lib.b200_conv_tma_weight_image_bytes(C.byref(d)) == p["image_bytes"], name
        assert lib.b200_conv_tma_workspace_bytes(C.byref(d)) == p["workspace_bytes"], name

    def some(pred):
        return any(pred(CASES[n], plans[n]) for n in CASES)

    assert {c["cout"] for c in CASES.values()} >= set(COUTS)
    assert {p["n_tile"] for p in plans.values()} == {64, 128, 256}
    assert {p["n_tiles_n"] for p in plans.values()} == {1, 2, 3}
    for n_tile, chunks, res in ((64, 12, True), (64, 13, False), (256, 3, True), (256, 4, False)):
        assert some(lambda c, p: (p["n_tile"], p["n_chunks"], p["resident"]) == (n_tile, chunks, res)), (n_tile, chunks)
    for n_tile, group in ((64, 4), (128, 2), (256, 1)):      # ragged last stage (nsub not a multiple of the group)
        assert some(lambda c, p: p["n_tile"] == n_tile and p["b_group"] == group and not p["resident"]
                    and (group == 1 or p["nsub"] % group)), (n_tile, group)
    for n_tile in (64, 128, 256):
        assert some(lambda c, p: p["n_tile"] == n_tile and p["total_tiles"] >= 3 * H100_SMS and p["n_chunks"] >= 50
                    and not p["resident"]), n_tile
    for cin, kw, folded in ((8, 7, True), (9, 7, False), (32, 2, True), (16, 3, True), (21, 3, False), (1, 3, True)):
        assert some(lambda c, p: (c["cin"], c["k"][1], p["fold_cf"] > 0) == (cin, kw, folded)), (cin, kw)
    assert some(lambda c, p: p["fold_cf"] and c["pad_mode"] == "reflect")
    assert some(lambda c, p: p["fold_cf"] and c["upsample"] == 2)
    assert some(lambda c, p: p["fold_cf"] and c["n"] > 1)
    assert some(lambda c, p: p["fold_cf"] and c["in_slice"] and c["in_slice"][0] % 2 == 1)
    assert all(p["fold_cf"] == 0 for n, p in plans.items() if CASES[n]["stride"] == 2)
    s2 = [c for c in CASES.values() if c["stride"] == 2]
    assert {c["k"] for c in s2} >= {(kh, kw) for kh in (1, 3) for kw in (1, 3, 4, 7)}
    assert all(c["h"] % 2 and c["w"] % 2 for c in s2 if c["upsample"] == 1)
    assert some(lambda c, p: c["stride"] == 2 and c["pad_mode"] == "reflect")
    assert some(lambda c, p: c["stride"] == 2 and c["upsample"] == 2 and c["up_mode"] == "nearest")
    for kw in (15, 31):
        assert some(lambda c, p: c["k"][1] == kw and c["stride"] == 1 and p["a_rows"] > 128)
    ragged = {p["ow"] for n, p in plans.items() if p["oh"] == 1 and CASES[n]["n"] == 3}
    assert ragged >= {1, 127, 128, 129, 255, 257}
    assert some(lambda c, p: (c["w"] + 2 * c["pad"][1]) % 32 != 0 and p["fold_cf"] == 0)
    for off in (3, 61):
        assert some(lambda c, p: c["in_slice"] and c["in_slice"][0] == off and c["cin"] % 16)
    assert some(lambda c, p: c["up_mode"] == "bilinear" and c["h"] == 1)
    assert some(lambda c, p: c["up_mode"] == "bilinear" and c["w"] == 1)
    assert some(lambda c, p: c["up_mode"] == "bilinear" and c["pad_mode"] == "reflect")
    assert some(lambda c, p: c["up_mode"] == "bilinear" and c["stride"] == 2)
    assert some(lambda c, p: c["pad_mode"] == "reflect" and c["pad"] == (c["h"] - 1, c["w"] - 1))
    assert {c["act"] for c in CASES.values()} == set(ACTS)
    assert some(lambda c, p: c["out_scale"] != 1.0 and c["res_slice"] is not None and c["res_slice"][0] > 0)
    assert some(lambda c, p: not c["bias"])
    assert some(lambda c, p: c["out_slice"] and c["out_slice"][0] > 0 and c["out_slice"][1] > c["out_slice"][0] + c["cout"])
    assert some(lambda c, p: c["saturate"])


def test_tma_chain_refuses_a_bad_residual_slice(lib):
    """b200_conv2d_tma_chain validates the residual channel slice before anything is launched (as b200_conv2d does).
    The pointers are host buffers: validation never dereferences them."""
    c = dict(CASES["residual_offset"])
    buf = torch.zeros(1 << 16)
    for off, total in ((11, 50), (-1, 50), (0, 39)):
        d = _desc(dict(c, res_slice=(off, total)))
        rc = lib.b200_conv2d_tma_chain(C.byref(d), N.ptr(buf), None, N.ptr(buf), N.ptr(buf), N.ptr(buf), N.ptr(buf), None,
                                       None, 0, N.ptr(buf), buf.numel() * 4, None)
        assert rc != 0 and b"residual slice out of range" in lib.b200_last_error(), (off, total)


def test_too_wide_filter_is_refused_by_the_planner(lib):
    """The activation box holds at most 256 pixel rows: KW 130 at stride 1 (259 at stride 2) has no workspace size and
    no weight image, so nothing is launched for it; KW 129 (258) is the widest accepted."""
    for stride, kw_ok in ((1, 129), (2, 258)):
        for kw, ok in ((kw_ok, True), (kw_ok + 1, False)):
            c = dict(CASES["abox_1x129"], k=(1, kw), pad=(0, kw // 2), stride=stride)
            d = _desc(c)
            ws, img = lib.b200_conv_tma_workspace_bytes(C.byref(d)), lib.b200_conv_tma_weight_image_bytes(C.byref(d))
            if ok:
                assert ws == plan(c)["workspace_bytes"] and img == plan(c)["image_bytes"], (stride, kw)
            else:
                assert ws == -1 and img == -1 and b"filter too wide" in lib.b200_last_error(), (stride, kw)
