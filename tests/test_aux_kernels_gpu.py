"""Kernel-level tests of the input producer (csrc/producer.cu), the RAFT correlation kernels (csrc/raft_kernels.cu,
the SIMT GEMM of csrc/mlp_simt.cu, the wgmma builder of csrc/conv_tma.cu) and the small image operators of
csrc/conv_simt.cu, each against a plain reference computed here on the CPU, at the shapes where such kernels go wrong:
odd and one-pixel planes, sizes that are not multiples of the vector width, channel slices of larger buffers,
coordinates on and beyond the borders.  The pipelines that use these kernels are tested end to end elsewhere, at a
few fixture sizes only.

Every test states its bound in its docstring and prints the measured error next to it (`pytest -s`).
u = 2^-24 is the unit roundoff of fp32."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from b200 import _native as N
from b200 import nn as K
from oracle import flow_oracle as FO
from oracle import loader_oracle as LO

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -24


def _report(what, err, bound):
    print(f"{what}: error {err:.3e}  bound {bound:.3e}")
    assert err <= bound, f"{what}: error {err:.3e} > bound {bound:.3e}"


# ---------------------------------------------------------------------------------------------------------------
# Input producer: bit for bit against oracle/loader_oracle.py (itself pinned against OpenCV)
# ---------------------------------------------------------------------------------------------------------------
def _flow_pair(f12, f21, H, W, T, first, records, bits_f, bits_b, t_begin=0, t_end=None, filt=1):
    lib = N.lib()
    h, w = f12.shape[:2]
    d12 = torch.from_numpy(np.ascontiguousarray(f12, dtype=np.float32)).to(DEV)
    d21 = torch.from_numpy(np.ascontiguousarray(f21, dtype=np.float32)).to(DEV)
    scratch = torch.empty(int(lib.b200_producer_scratch_floats(H, W)), dtype=torch.float32, device=DEV)
    N.check(lib.b200_producer_flow_pair(N.ptr(d12), N.ptr(d21), h, w, H, W, T, t_begin, T if t_end is None else t_end,
                                        N.ptr(records), N.ptr(bits_f), N.ptr(bits_b), first, filt, N.ptr(scratch),
                                        N.current_stream()), "b200_producer_flow_pair")
    torch.cuda.synchronize()


def _video_buffers(H, W, T, frames):
    records = torch.zeros(max(H * W * frames, 1) * N.RECORD_FLOATS, dtype=torch.float32, device=DEV)
    words = (H * W * T + 31) // 32 + 1             # a warp whose pixels straddle the last word ORs into one more
    return records, torch.zeros(words, dtype=torch.int32, device=DEV), torch.zeros(words, dtype=torch.int32, device=DEV)


# (h, w) of the RAFT flow -> (H, W) of the atlas
RESIZE_GEOMETRIES = {
    "half_both_area_path": (60, 88, 30, 44),
    "half_height_only": (60, 57, 30, 44),
    "half_height_same_width": (60, 44, 30, 44),
    "integer_factor_4": (120, 176, 30, 44),
    "fractional": (47, 71, 29, 43),
    "width_only_half": (30, 88, 30, 44),
    "width_only_fractional": (30, 61, 30, 44),
    "identity": (29, 43, 29, 43),
}


@pytest.mark.parametrize("name", list(RESIZE_GEOMETRIES))
def test_producer_resize_is_bit_exact(name):
    """Flows resized on the device (cv2.resize INTER_LINEAR, OpenCV's area-fast path at exactly half size, the
    reference's swapped scale factors; no resize launch at equal size) against loader_oracle.resize_flow: bit for bit."""
    h, w, H, W = RESIZE_GEOMETRIES[name]
    rng = np.random.default_rng(h * 1000 + w)
    f12 = (rng.standard_normal((h, w, 2)) * 7).astype(np.float32)
    f21 = (rng.standard_normal((h, w, 2)) * 7).astype(np.float32)
    records, bf, bb = _video_buffers(H, W, 2, 2)
    _flow_pair(f12, f21, H, W, 2, 0, records, bf, bb, filt=0)
    rec = records.view(2, H, W, N.RECORD_FLOATS).cpu()
    want12 = torch.from_numpy(LO.resize_flow(f12, H, W))
    want21 = torch.from_numpy(LO.resize_flow(f21, H, W))
    n_diff = int((rec[0, :, :, 9:11] != want12).sum() + (rec[1, :, :, 11:13] != want21).sum())
    print(f"resize {name} {h}x{w} -> {H}x{W}: {n_diff} values differ (bound 0)")
    assert torch.equal(rec[0, :, :, 9:11], want12)
    assert torch.equal(rec[1, :, :, 11:13], want21)
    # filter off: every frame with a partner is valid (unwrap_utils.py:160-162), the others stay zero
    assert torch.all(rec[0, :, :, 13] == 1) and torch.all(rec[1, :, :, 14] == 1)
    assert torch.all(rec[0, :, :, 14] == 0) and torch.all(rec[1, :, :, 13] == 0)


def _edge_flows(H, W, seed):
    """A smooth forward flow with a nearly consistent backward flow (so that both mask values occur), overwritten
    in places with what the consistency kernel's edge cases need."""
    rng = np.random.default_rng(seed)
    ys, xs = np.mgrid[0:H, 0:W].astype(np.float32)
    f12 = np.stack([2.0 * np.sin(ys / 3.0 + xs / 5.0), 1.5 * np.cos(xs / 4.0)], -1).astype(np.float32)
    # sampling coordinates in (-1, 0) on the first row / column: the 1/32 grid index is negative and `>> 5` floors
    f12[:, 0, 0] = -rng.uniform(0.01, 0.99, H)
    f12[0, :, 1] = -rng.uniform(0.01, 0.99, W)
    # taps across the last row / column (the +1 taps fall outside)
    f12[:, W - 1, 0] = rng.uniform(0.01, 0.99, H)
    f12[H - 1, :, 1] = rng.uniform(0.01, 0.99, W)
    # exact 1/64-pixel offsets: 32 * coordinate is a half integer, rounded half to even
    k = rng.choice(np.arange(-15, 16, 2), size=(3, 6, 2))
    f12[2:5, 3:9] = (k / 64.0).astype(np.float32)
    # flows larger than the frame, in both directions
    f12[5, :, 0] = np.where(np.arange(W) % 2 == 0, W + 3.3, -(2 * W + 0.7))
    f12[6, :, 1] = np.where(np.arange(W) % 3 == 0, H + 0.4, -(3 * H + 1.6))
    f12[7, 1:4] = [[1.0e4, -2.5e3], [-7.7e3, 9.1e3], [0.5, -1.0e4]]
    f21 = (-f12 + rng.normal(0, 0.7, f12.shape)).astype(np.float32)
    f21[:, 0] = rng.normal(0, 4.0, (H, 2))                 # large values right at the border taps
    f21[H - 1] = rng.normal(0, 4.0, (W, 2))
    return f12, f21.astype(np.float32)


def _want_masks(f12, f21):
    return LO.consistency_error(f12, f21) < 1.0, LO.consistency_error(f21, f12) < 1.0


@pytest.mark.parametrize("H,W", [(13, 19), (17, 37), (9, 9)])
def test_producer_consistency_and_bitmaps_are_bit_exact(H, W):
    """Consistency masks (cv2.remap of the partner flow on the 1/32 grid, zero border, |.| < 1) of a 3-frame video
    whose H*W is not a multiple of 32, so pair offsets straddle bitmap words: record slots 9..14 and both whole-video
    bitmaps against loader_oracle, bit for bit, for the whole video resident and for two frame shards — one of
    them holds neither frame of the first pair (records = NULL, only the bitmaps are written)."""
    T = 3
    HW = H * W
    assert HW % 32
    pairs = [_edge_flows(H, W, seed) for seed in range(T - 1)]
    masks = [_want_masks(f12, f21) for f12, f21 in pairs]
    fwd = np.zeros((T, HW), bool)
    bwd = np.zeros((T, HW), bool)
    for i, (mf, mb) in enumerate(masks):
        fwd[i] = mf.reshape(-1)
        bwd[i + 1] = mb.reshape(-1)
    assert 0.05 < fwd[:T - 1].mean() < 0.95 and 0.05 < bwd[1:].mean() < 0.95          # both mask values occur
    words = (HW * T + 31) // 32 + 1

    def packed(m):
        b = np.zeros(words * 32, bool)
        b[:HW * T] = m.reshape(-1)
        return torch.from_numpy(np.packbits(b, bitorder="little").view(np.int32).copy())

    for t_begin, t_end in ((0, T), (1, 2), (2, 3)):
        records, bf, bb = _video_buffers(H, W, T, t_end - t_begin)
        for i, (f12, f21) in enumerate(pairs):
            resident = (t_begin <= i < t_end) or (t_begin <= i + 1 < t_end)
            _flow_pair(f12, f21, H, W, T, i, records if resident else None, bf, bb, t_begin, t_end)
        assert torch.equal(bf.cpu(), packed(fwd)), (t_begin, t_end)
        assert torch.equal(bb.cpu(), packed(bwd)), (t_begin, t_end)
        rec = records.view(t_end - t_begin, HW, N.RECORD_FLOATS).cpu()
        for t in range(t_begin, t_end):
            r = rec[t - t_begin]
            want_f = torch.from_numpy(fwd[t].astype(np.float32))
            want_b = torch.from_numpy(bwd[t].astype(np.float32))
            assert torch.equal(r[:, 13], want_f) and torch.equal(r[:, 14], want_b), (t_begin, t_end, t)
            if t < T - 1:
                assert torch.equal(r[:, 9:11], torch.from_numpy(pairs[t][0]).reshape(HW, 2))
            if t > 0:
                assert torch.equal(r[:, 11:13], torch.from_numpy(pairs[t - 1][1]).reshape(HW, 2))
    print(f"consistency {H}x{W}: masks and bitmaps bit-exact (bound: exact); "
          f"forward valid {fwd[:T - 1].mean():.2f}, backward valid {bwd[1:].mean():.2f}")


def test_producer_consistency_on_resized_flows():
    """The consistency kernel on flows the device resized (fractional factor): masks == oracle masks of the
    oracle-resized flows, bit for bit."""
    H, W = 21, 30
    big = [_edge_flows(35, 47, 5)]
    f12 = LO.resize_flow(big[0][0], H, W)
    f21 = LO.resize_flow(big[0][1], H, W)
    mf, mb = _want_masks(f12, f21)
    records, bf, bb = _video_buffers(H, W, 2, 2)
    _flow_pair(big[0][0], big[0][1], H, W, 2, 0, records, bf, bb)
    rec = records.view(2, H * W, N.RECORD_FLOATS).cpu()
    assert torch.equal(rec[0, :, 13], torch.from_numpy(mf.reshape(-1).astype(np.float32)))
    assert torch.equal(rec[1, :, 14], torch.from_numpy(mb.reshape(-1).astype(np.float32)))
    print(f"consistency on resized flows: bit-exact (bound: exact), valid {mf.mean():.2f} / {mb.mean():.2f}")


@pytest.mark.parametrize("H,W", [(13, 19), (1, 37), (23, 1), (1, 1)])
def test_producer_frame_kernel(H, W):
    """rgb and the forward differences (np.diff semantics, zero in the last column / row) of one frame, bit for bit;
    the flow and mask slots of the record are left alone."""
    rng = np.random.default_rng(H * 100 + W)
    frame = rng.random((H, W, 3)).astype(np.float32)
    dev = torch.from_numpy(frame).to(DEV).reshape(-1)
    rec = torch.full((H * W * N.RECORD_FLOATS,), -3.0, dtype=torch.float32, device=DEV)
    N.check(N.lib().b200_producer_frame(N.ptr(dev), H, W, N.ptr(rec), N.current_stream()), "b200_producer_frame")
    rec = rec.view(H, W, N.RECORD_FLOATS).cpu()
    dx = np.zeros_like(frame)
    dy = np.zeros_like(frame)
    dx[:, :-1] = np.diff(frame, axis=1)
    dy[:-1] = np.diff(frame, axis=0)
    assert torch.equal(rec[..., 0:3], torch.from_numpy(frame))
    assert torch.equal(rec[..., 3:6], torch.from_numpy(dx))
    assert torch.equal(rec[..., 6:9], torch.from_numpy(dy))
    assert torch.all(rec[..., 9:] == -3.0)
    print(f"frame kernel {H}x{W}: bit-exact (bound: exact)")


@pytest.mark.parametrize("h,w", [(29, 44), (30, 43), (12, 20)])
def test_producer_rejects_upscaling(h, w):
    """A flow smaller than the working resolution in either dimension is refused (the host resizes it instead)."""
    H, W = 30, 44
    records, bf, bb = _video_buffers(H, W, 2, 2)
    f = np.zeros((h, w, 2), np.float32)
    with pytest.raises(N.B200Error, match="covers down-scaling only"):
        _flow_pair(f, f, H, W, 2, 0, records, bf, bb)


# ---------------------------------------------------------------------------------------------------------------
# Correlation pyramid and lookup
# ---------------------------------------------------------------------------------------------------------------
def _levels(flat, H8, W8):
    out, off, h, w = [], 0, H8, W8
    for _ in range(4):
        n = H8 * W8 * h * w
        out.append(flat[off:off + n].view(H8 * W8, 1, h, w))
        off += n
        h //= 2
        w //= 2
    assert off == flat.numel()
    return out


def _fmaps(dim, H8, W8, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(1, dim, H8, W8, generator=g), torch.randn(1, dim, H8, W8, generator=g)


# max error / max|level| of the pyramid, in units of u * sqrt(dim): fp32 dot products of `dim` terms
CORR_BUILD_BOUND = {"simt": 4.0, "tc": 8.0}


@pytest.mark.parametrize("impl", ["simt", "tc"])
@pytest.mark.parametrize("dim", [256, 96])
@pytest.mark.parametrize("H8,W8", [(8, 8), (9, 11), (13, 37), (17, 130)])
def test_corr_build(H8, W8, dim, impl):
    """Every pyramid level (the coarsest one 1 pixel high or wide for H8 or W8 < 16; H8*W8 not a multiple of 4 runs
    the SIMT GEMM's scalar loads) against float64 matmul / sqrt(dim) + avg_pool2d.  The rounding error of an fp32
    dot product of `dim` terms grows like u sqrt(dim) relative to max|level|: bound 4 u sqrt(dim) * max|level| for
    the fp32 CUDA-core GEMM, 8 u sqrt(dim) * max|level| for the wgmma builder, whose split fp16 operands also drop
    the lo * lo products (2^-22 relative).  Measured on an H100 80GB HBM3 (400 W): at most 0.19 of the bound."""
    f1, f2 = _fmaps(dim, H8, W8, H8 * 1000 + W8 + dim)
    HW = H8 * W8
    lvl = (f1.double().view(dim, HW).t() @ f2.double().view(dim, HW) / math.sqrt(dim)).view(HW, 1, H8, W8)
    want = [lvl]
    for _ in range(3):
        want.append(F.avg_pool2d(want[-1], 2, stride=2))
    got = _levels(K.corr_build(f1.to(DEV), f2.to(DEV), impl=impl).cpu().double(), H8, W8)
    for l, (g, r) in enumerate(zip(got, want)):
        assert g.shape == r.shape
        _report(f"corr_build[{impl}] {H8}x{W8} dim {dim} level {l}", ((g - r).abs().max() / r.abs().max()).item(),
                CORR_BUILD_BOUND[impl] * U * math.sqrt(dim))


def _lookup_coords(H8, W8, seed):
    g = torch.Generator().manual_seed(seed)
    ys, xs = torch.meshgrid(torch.arange(H8, dtype=torch.float32), torch.arange(W8, dtype=torch.float32), indexing="ij")
    c = torch.stack([xs, ys]) + (torch.rand(2, H8, W8, generator=g) - 0.5) * 6.0
    flat = c.view(2, -1)
    n = flat.shape[1]
    idx = torch.randperm(n, generator=g)
    special = [(float(i % W8), float(i // W8)) for i in range(0, n, 7)][:8]           # integer pixel centres
    special += [(W8 - 1.0, H8 - 1.0), (W8 - 1.0, 2.0), (3.0, H8 - 1.0), (W8 - 1.25, H8 - 0.75)]   # last row / column
    special += [(-2.5, 1.0), (W8 + 1.7, H8 + 0.3), (-0.4, -3.2), (W8 + 4.0, -1.0)]    # a few pixels outside
    special += [(1e3, 2.0), (-1e3, 1.0), (3.0, 1e3), (2.0, -1e3)]                    # far outside the staged window
    special += [(1e7, 1.0), (-1e7, -1e7), (5.0, 1e7), (1e7, -1e7)]                   # clamped window origin
    for k, (x, y) in enumerate(special):
        flat[0, idx[k]], flat[1, idx[k]] = x, y
    return c.unsqueeze(0).contiguous()


@pytest.mark.parametrize("H8,W8", [(9, 11), (13, 37), (17, 130)])
def test_corr_lookup_all_radii(H8, W8):
    """Radius 1..8 (the shared-memory tiled kernel for r <= 4, the plain kernel above) against
    flow_oracle.corr_lookup in float64 on the device's own pyramid; coordinates on pixel centres, on the last row /
    column, a few pixels outside, at +-1e3 and +-1e7.  The error is dominated by the sampling coordinate, not by the
    bilinear arithmetic: the reference's fp32 round trip x -> 2x/(W-1) - 1 -> ((g+1)/2)(W-1) moves it by a few
    u (W + H) pixels at the level's size.  Bound per level over the finite outputs: 2 u (W_l + H_l) * max|level_l|
    (measured on an H100 80GB HBM3 (400 W): at most 0.38 of it; 6.7e-6 * max|level| at 17x130).  A level 1 pixel
    high or wide makes the reference's normalised coordinates non-finite: the output is NaN exactly where the
    oracle's is (the whole level)."""
    f1, f2 = _fmaps(64, H8, W8, 7 * H8 + W8)
    pyr = K.corr_build(f1.to(DEV), f2.to(DEV), impl="simt")
    levels = [p.double() for p in _levels(pyr.cpu(), H8, W8)]
    coords = _lookup_coords(H8, W8, H8 + W8)
    errs = {}
    for r in range(1, 9):
        taps = (2 * r + 1) ** 2
        got = K.corr_lookup(pyr, coords.to(DEV), r).cpu().double()
        want = FO.corr_lookup(levels, coords.double(), radius=r).double()
        assert got.shape == want.shape == (1, 4 * taps, H8, W8)
        assert torch.equal(torch.isnan(got), torch.isnan(want)), f"radius {r}: NaN pattern differs"
        for l in range(4):
            g, w = got[:, l * taps:(l + 1) * taps], want[:, l * taps:(l + 1) * taps]
            if levels[l].shape[-1] == 1 or levels[l].shape[-2] == 1:
                assert torch.isnan(g).all(), f"radius {r} level {l}"
                continue
            assert torch.isfinite(g).all()
            errs[(r, l)] = ((g - w).abs().max() / levels[l].abs().max()).item() / (2 * U * sum(levels[l].shape[-2:]))
    for l in range(4):
        row = [f"{errs[(r, l)]:.3f}" for r in range(1, 9) if (r, l) in errs]
        if row:
            print(f"corr_lookup {H8}x{W8} level {l} {tuple(levels[l].shape[-2:])}, error / bound for radius 1..8: "
                  f"{' '.join(row)}")
    _report(f"corr_lookup {H8}x{W8} worst error / bound", max(errs.values()), 1.0)


# ---------------------------------------------------------------------------------------------------------------
# Image operators of conv_simt.cu against float64 torch
# ---------------------------------------------------------------------------------------------------------------
IN_SHAPES = [(2, 3, 1, 1), (1, 4, 1, 3), (2, 2, 7, 13), (1, 3, 20, 50), (1, 2, 33, 65), (1, 2, 512, 515),
             (1, 2, 513, 515)]


@pytest.mark.parametrize("relu", [False, True])
@pytest.mark.parametrize("shape", IN_SHAPES)
def test_instance_norm(shape, relu):
    """nn.InstanceNorm2d (eps 1e-5, no affine) +- ReLU against float64, planes of 1, 3, 91, 1000, 2145, 263680 and
    263695 pixels (float4 loads only when H*W % 4 == 0, scalar loads otherwise; fewer and more pixels than the 1024
    threads), plane means up to 10 standard deviations, one constant plane (output exactly 0).
    Bound per plane: y = (x - mean) / std is rounded twice per element (2 u of |mean| / std + |y|); the fp32 mean
    and centred variance are sums of hw terms (ceil(hw / 1024) per thread, then a 10-level tree) whose rounding
    errors partly cancel and, scaled by 1 / std, add a few u |mean| / std:
    |dy| <= 6 u (|mean| / std + max|y| + 1).  Measured on an H100 80GB HBM3 (400 W): at most 0.17 of it."""
    n, c, h, w = shape
    g = torch.Generator().manual_seed(h * 7919 + w)
    planes = n * c
    ratio = torch.linspace(0.0, 10.0, planes).view(n, c, 1, 1)         # |mean| / std per plane
    std = torch.logspace(-2, 2, planes).view(n, c, 1, 1)
    sign = torch.where(torch.arange(planes).view(n, c, 1, 1) % 2 == 0, 1.0, -1.0)
    x = torch.randn(n, c, h, w, generator=g) * std + sign * ratio * std
    if h * w > 1:
        x[0, 0] = 2.5                                                        # constant plane
    y = K.instance_norm(x.to(DEV), relu=relu).cpu().double()
    xd = x.double()
    mean = xd.mean(dim=(2, 3), keepdim=True)
    var = ((xd - mean) ** 2).mean(dim=(2, 3), keepdim=True)
    ref = (xd - mean) / torch.sqrt(var + 1e-5)                  # F.instance_norm refuses 1-pixel planes
    if relu:
        ref = torch.relu(ref)
    if h * w > 1:
        assert torch.all(y[0, 0] == 0), "a constant plane normalises to 0"
    sd = var.sqrt().clamp_min(1e-30)
    scale = (mean.abs() / sd).amax(dim=(2, 3)).clamp_max(1e3) + ref.abs().amax(dim=(2, 3)) + 1.0
    bound = 6 * U * scale
    err = (y - ref).abs().amax(dim=(2, 3))
    ratio_used = (err / bound).max().item()
    print(f"instance_norm {shape} relu={relu}: max error {err.max().item():.3e}, worst error / bound {ratio_used:.3f}")
    assert ratio_used <= 1.0


@pytest.mark.parametrize("h,w", [(5, 7), (9, 2), (2, 11), (33, 65), (2, 2)])
def test_maxpool2(h, w):
    """nn.MaxPool2d(2, 2) (floor mode: the last odd row / column is dropped): torch.equal with F.max_pool2d."""
    g = torch.Generator().manual_seed(h * 31 + w)
    x = torch.randn(2, 3, h, w, generator=g)
    y = K.maxpool2(x.to(DEV)).cpu()
    assert torch.equal(y, F.max_pool2d(x, 2, 2))
    print(f"maxpool2 {h}x{w}: exact (bound: exact)")


@pytest.mark.parametrize("h,w", [(1, 1), (1, 9), (7, 1), (5, 7), (17, 33)])
def test_upsample_bilinear2_into_channel_slice(h, w):
    """nn.Upsample(2, bilinear, align_corners=True) written into channels [2, 2 + C) of a larger buffer filled with a
    sentinel: the other channels keep it; the slice matches F.interpolate in float64 within
    2 u (H + W + 2) max|x|: the fp32 source coordinate dst * (in-1)/(out-1) is off by up to u * in pixels per axis,
    and neighbouring inputs differ by up to 2 max|x|."""
    n, c, extra = 2, 3, 4
    g = torch.Generator().manual_seed(h * 13 + w)
    x = torch.randn(n, c, h, w, generator=g)
    out = torch.full((n, c + extra, 2 * h, 2 * w), 1234.5, device=DEV)
    K.upsample_bilinear2(x.to(DEV), out=out, out_c_off=2)
    out = out.cpu()
    ref = F.interpolate(x.double(), scale_factor=2, mode="bilinear", align_corners=True)
    assert torch.all(out[:, :2] == 1234.5) and torch.all(out[:, 2 + c:] == 1234.5), "channels outside the slice"
    bound = 2 * U * (h + w + 2) * x.abs().max().item()
    _report(f"upsample_bilinear2 {h}x{w}", (out[:, 2:2 + c].double() - ref).abs().max().item(), bound)


def test_gru_gate_both_modes():
    """mode 0 (r * h) into the first C channels of a concat buffer, the other channels untouched: exactly the fp32
    product.  mode 1 ((1 - z) h + z q) against float64 within 4 u max(|h|, |q|)."""
    g = torch.Generator().manual_seed(21)
    n, c, h, w, c_total = 2, 5, 7, 9, 12
    a = torch.sigmoid(torch.randn(n, c, h, w, generator=g) * 3)
    b = torch.randn(n, c, h, w, generator=g) * 2
    q = torch.tanh(torch.randn(n, c, h, w, generator=g))
    buf = torch.full((n, c_total, h, w), -7.25, device=DEV)
    K.gru_gate(a.to(DEV), b.to(DEV), out=buf, mode=0)
    buf = buf.cpu()
    assert torch.equal(buf[:, :c], a * b)
    assert torch.all(buf[:, c:] == -7.25)
    got = K.gru_gate(a.to(DEV), b.to(DEV), q.to(DEV), mode=1).cpu().double()
    ref = (1 - a.double()) * b.double() + a.double() * q.double()
    bound = 4 * U * max(b.abs().max().item(), q.abs().max().item())
    _report("gru_gate mode 1", (got - ref).abs().max().item(), bound)


@pytest.mark.parametrize("shape", [(2, 3, 5, 7), (1, 1, 1, 1), (1, 8, 16, 24)])
def test_convlstm_zero_state(shape):
    """ConvLSTM step from a zero state: hidden = sigmoid(o) tanh(sigmoid(i) tanh(g)), cell = sigmoid(i) tanh(g),
    against float64 within 1e-6 (outputs in (-1, 1); expf / tanhf are accurate to a few ulp).  Without a cell
    tensor the hidden state is bit-identical."""
    n, c, h, w = shape
    g = torch.Generator().manual_seed(n * 100 + c)
    gates = torch.randn(n, 4 * c, h, w, generator=g) * 4
    hid, cell = K.convlstm_zero_state(gates.to(DEV), want_cell=True)
    hid2, none = K.convlstm_zero_state(gates.to(DEV), want_cell=False)
    assert none is None and torch.equal(hid, hid2)
    gd = gates.double()
    i_g, _, o_g, c_g = gd.chunk(4, 1)
    ref_cell = torch.sigmoid(i_g) * torch.tanh(c_g)
    ref_hid = torch.sigmoid(o_g) * torch.tanh(ref_cell)
    _report(f"convlstm {shape} hidden", (hid.cpu().double() - ref_hid).abs().max().item(), 1e-6)
    _report(f"convlstm {shape} cell", (cell.cpu().double() - ref_cell).abs().max().item(), 1e-6)


@pytest.mark.parametrize("numel", [1, 255, 257, 3 * 5 * 7 * 11])
def test_add_relu(numel):
    """relu(a + b): exactly the fp32 sum."""
    g = torch.Generator().manual_seed(numel)
    a, b = torch.randn(numel, generator=g), torch.randn(numel, generator=g)
    got = K.add_relu(a.to(DEV), b.to(DEV)).cpu()
    assert torch.equal(got, torch.relu(a + b))
    print(f"add_relu {numel}: exact (bound: exact)")


@pytest.mark.parametrize("h,w", [(5, 7), (1, 1), (3, 1), (6, 9)])
def test_convex_upsample(h, w):
    """RAFT convex 8x upsampling, N = 2, mask logits up to +-80 (a softmax without the max shift overflows),
    against flow_oracle.convex_upsample in float64 within 8 u * 8 max|flow| (nine fp32 weights and products,
    accumulated in fp32)."""
    n = 2
    g = torch.Generator().manual_seed(h * 10 + w)
    flow = torch.randn(n, 2, h, w, generator=g) * 5
    mask = (torch.rand(n, 576, h, w, generator=g) * 2 - 1) * 80
    got = K.convex_upsample(flow.to(DEV), mask.to(DEV)).cpu().double()
    ref = FO.convex_upsample(flow.double(), mask.double())
    assert torch.isfinite(got).all()
    bound = 8 * U * 8 * flow.abs().max().item()
    _report(f"convex_upsample {h}x{w}", (got - ref).abs().max().item(), bound)
