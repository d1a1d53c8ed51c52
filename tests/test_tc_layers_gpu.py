"""The fused tensor-core IMLP kernels of csrc/mlp_tc.cu (tc_prep_kernel, tc_fwd_kernel, tc_bwd_kernel, tc_wgrad_kernel)
one layer at a time against float64 references built from the operands the kernels themselves read.

Each case runs a training forward and a backward, then decodes the operand images the kernels left in the workspace:
the split weight items (W for the forward, W^T for the dgrad), the forward constants, every activation image, the
ReLU flag words, the positional-encoding image, every dZ image and the output layer's dZ image.
b200_mlp_tc_image_offsets / b200_atlas_tc_image_offsets_for locate them, and `atom_off`, `tile_off` and `item_off`
in tc_images_common.py mirror the kernels' swizzles.

(a) Weight images and forward constants, bit for bit: hi = rn_f16(256 W), lo = rn_f16(256 W - hi), both saturating
    (cvt.rn.satfinite), in the chunk order hi k0-31, hi k32-63, lo k0-31, lo k32-63, zero outside the weight; the
    constants are the fp32 products of DESIGN §4.
(b)-(d) Every other value v is compared with v64, the float64 evaluation of the same operation on the device's own
    split operands: the three products hi*hi + hi*lo + lo*hi of the previous image and the weight items, masked by
    the device's own flag bits.  No ReLU mask is recomputed, so no mask can flip between the two sides.  Per element,
    with u = 2^-24 and c = 4:

        |v - v64| <= c u (sqrt(K) + chain) A + 2^-22 |v64| + 2^-24

    A      the float64 sum of |products| (and |bias|) of the element, in the image's scaled units
    K      the reduction length: 256 (hidden layers), 64 / 320 with the encoding chunk, the output layer's 256 / 296
           columns; for dW the most rows one unit of the work list sums (its share of the live tiles)
    chain  one fp32 rounding per wgmma that accumulates into the element (3 per 16 of K) plus one in the epilogue;
           CUDA-core layers: one per sequential fma of a thread (K / 4 + 3 for the output layer, 3 for the plain
           mapping's layer 0); dW: 3 per 16 rows plus one fp32 atomic per unit (both CTAs of a pair flush)
    2^-22 |v64| + 2^-24   the 2-term split of the result (22 significand bits, fp16 subnormal floor)

    Where |z64| of a pre-activation exceeds its bound the flag must equal z64 > 0, and a zero flag must come with an
    exactly zero image.  The encoding is held to 4u of float64 sin / cos of the fp32 products x b_k (sinf / cosf are
    within 2 ulp), tanhf to 4u |y|, the output dZ image to dy (1 - y^2) with the device's y, and the gradient scale
    s_g is recomputed from the gmax word the call used with the rule of `grad_scales`.

Cases: the stand-alone `IMLP` call for the six networks with tensor-core kernels at the row counts of
test_wgrad_gpu.py and test_bwd_reductions_gpu.py (1, 127, 129, one tile per cluster of two SMs less / more one tile,
3 * 132 * 128 - 50), and the fused stage-1 step at 80 x 432 x 768 with B = 10 000, with and without the global
rigidity term (nine or seven mapping groups, the two flow-match groups compacted to their valid rows, one work list for
both networks).  The atlas input gradient is checked in the stand-alone calls, where the kernel overwrites it (in the
step it is added to the loss head's).  Bias gradients and the plain mapping's dW0 are test_bwd_reductions_gpu.py's.
Each case prints its largest ratio of error to bound (`pytest -s`).
"""
import ctypes as C
import math
import os
import zlib

import numpy as np
import pytest
import torch

from b200 import _native as N
from b200 import atlas as A
from b200 import synth
from oracle import atlas_oracle as O
from tc_images_common import (DEV, GMAX, OFFSETS, TM, Images, Net, Worst, check_backward, check_forward,
                              check_input_gradient, check_weight_gradients, check_weight_images, grad_scale, unit_splits,
                              wg_units, wgrad_gemms)  # noqa: F401  (wg_units: a fixture)

pytestmark = pytest.mark.gpu

# name: (input_dim, output_dim, num_layers, pe_freqs, skips), input scale, input shift
NETS = {
    "mapping": ((3, 2, 6, 0, ()), 2.0, -1.0),
    "mapping4": ((3, 2, 4, 0, ()), 2.0, -1.0),
    "atlas": ((2, 3, 8, 10, (4, 7)), 1.0, 0.0),
    "alpha": ((3, 1, 8, 5, ()), 2.0, -1.0),
    "pe6": ((3, 2, 6, 4, ()), 2.0, -1.0),
    "pe4": ((3, 2, 4, 10, ()), 2.0, -1.0),
}
SMS = 132


def _cluster_rows():
    tiles = (torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else SMS) // 2
    return [128 * (tiles - 1) - 5, 128 * (tiles + 1) + 3]


ROWS = [1, 127, 129] + _cluster_rows() + [3 * SMS * 128 - 50]


# ---------------------------------------------------------------------------------------------------------------
# cases
# ---------------------------------------------------------------------------------------------------------------
def _seed(text):
    return zlib.crc32(text.encode()) & 0x7FFFFFFF


def _init_flat(net, g):
    """nn.Linear's default init ranges: weights and biases uniform in +-1/sqrt(fan_in)."""
    flat = torch.zeros(net.total)
    for i, (k, n) in enumerate(net.dims):
        flat[net.w_off[i]:net.w_off[i] + k * n] = (torch.rand(n * k, generator=g) * 2 - 1) / math.sqrt(k)
        flat[net.b_off[i]:net.b_off[i] + n] = (torch.rand(n, generator=g) * 2 - 1) / math.sqrt(k)
    return flat.to(DEV)


@pytest.mark.parametrize("rows", ROWS)
@pytest.mark.parametrize("which", list(NETS))
def test_imlp_layers(which, rows, wg_units):
    """The stand-alone IMLP call (b200_mlp_forward / backward at B200_PREC_TC): checks (a) to (d)."""
    lib = N.lib()
    dims, xs, xo = NETS[which]
    g = torch.Generator().manual_seed(_seed(f"{which}/{rows}"))
    net = Net(dims, None)
    net.flat = _init_flat(net, g)
    x = (torch.rand(rows, net.in_dim, generator=g) * xs + xo).to(DEV)
    dy = torch.randn(rows, net.out, generator=g).to(DEV)
    nbytes = int(lib.b200_mlp_workspace_bytes(C.byref(net.desc), rows, 1))
    ws = torch.full((nbytes,), 0xFF, dtype=torch.uint8, device=DEV)     # NaN in every unwritten float / fp16 pair
    y = torch.empty(rows, net.out, device=DEV)
    grads = torch.zeros(net.total, device=DEV)
    d_in = torch.full((rows, net.in_dim), float("nan"), device=DEV) if net.atlas else None
    st = N.current_stream()
    N.check(lib.b200_mlp_forward(C.byref(net.desc), N.ptr(net.flat), N.ptr(x), N.ptr(y), rows, 1, N.PREC_TC, N.ptr(ws),
                                 nbytes, st), "forward")
    N.check(lib.b200_mlp_backward(C.byref(net.desc), N.ptr(net.flat), N.ptr(x), N.ptr(dy), N.ptr(grads), N.ptr(d_in),
                                  rows, N.PREC_TC, N.ptr(ws), nbytes, st), "backward")
    torch.cuda.synchronize()
    off = (C.c_int64 * OFFSETS)()
    N.check(lib.b200_mlp_tc_image_offsets(C.byref(net.desc), rows, N.ptr(ws), off), "image offsets")
    rows_pad = -(-rows // TM) * TM
    assert off[11] == rows_pad and (off[5] >= 0) == (net.pe > 0)
    im = Images(ws, off, net, range(rows_pad // TM))
    word = int(ws[off[GMAX]:off[GMAX] + 8].view(torch.int32)[1 if net.out == 2 else 0])
    assert word == int(dy.abs().max().view(torch.int32)), "the gmax word is not max |dy|"
    s_g = grad_scale(word)
    pad = rows_pad - rows
    inp = torch.nn.functional.pad(x, (0, 0, 0, pad))
    y_pad = torch.nn.functional.pad(y, (0, 0, 0, pad))
    dy_pad = torch.nn.functional.pad(dy, (0, 0, 0, pad))
    worst = Worst()
    check_weight_images(im, net, worst)
    check_forward(im, net, inp, y_pad, worst, y_rows=rows)
    check_backward(im, net, y_pad, dy_pad, s_g, worst)
    if net.atlas:
        check_input_gradient(im, net, s_g, d_in, worst)
    gemms = wgrad_gemms(net)
    n_split = unit_splits([(a, b, 1) for _, a, b in gemms], wg_units)
    check_weight_gradients(im, net, grads, s_g, rows_pad // TM, n_split, worst)
    worst.report(f"{which} rows {rows}")


@pytest.mark.parametrize("with_global", [True, False])
def test_fused_step_layers(golden_dir, with_global, wg_units):
    """The fused stage-1 step at the benchmark shape: both networks, live tiles only."""
    lib = N.lib()
    H, W, T, B = 432, 768, 80, 10000
    data = synth.throughput_set(H, W, T, seed=0)
    z = np.load(os.path.join(golden_dir, "params_seed1234.npz"))
    vid = A.DeviceVideo.from_reference_layout(data, DEV)
    tr = A.AtlasTrainer(vid, {"samples_batch": B}, precision=N.PREC_TC, device=DEV)
    tr.load_state(O.state_dict_of([torch.from_numpy(z[f"map{i}"]) for i in range(12)]),
                  O.state_dict_of([torch.from_numpy(z[f"atl{i}"]) for i in range(16)]))
    tr.indices.copy_(torch.randint(H * W * T, (B,), generator=torch.Generator().manual_seed(1)))
    tr.loss_grad(with_global)
    torch.cuda.synchronize()
    cfg = tr._config(True)
    ws = tr._workspace()
    wo = (C.c_int64 * 8)()
    N.check(lib.b200_atlas_workspace_offsets_for(C.byref(cfg), C.byref(tr.map_desc), N.ptr(ws), wo), "offsets")
    cap = (B + TM - 1) // TM * TM
    ct = cap // TM
    cnt = [int(v) for v in ws[wo[0]:wo[0] + 32].view(torch.int32).cpu()]
    f32 = lambda o, n, w: ws[o:o + 4 * n * w].view(torch.float32).view(n, w)
    ng = 9 if with_global else 7
    map_tiles, atl_tiles = [], []
    for grp in range(ng):
        n = cnt[5] if grp == 5 else (cnt[6] if grp == 6 else cnt[0])
        map_tiles += [grp * ct + t for t in range(min(ct, -(-n // TM)))]
    for grp in range(3):
        atl_tiles += [grp * ct + t for t in range(min(ct, -(-cnt[0] // TM)))]
    assert cnt[5] < cnt[0] and cnt[6] < cnt[0] and (cnt[5] % TM or cnt[6] % TM)
    rows_of = lambda tiles: (torch.as_tensor(tiles, device=DEV)[:, None] * TM + torch.arange(TM, device=DEV)).flatten()
    x_map, d_uv, uv = f32(wo[2], 9 * cap, 4), f32(wo[4], 9 * cap, 2), f32(wo[6], 9 * cap, 2)
    d_y, y_atl = f32(wo[5], 3 * cap, 3), f32(wo[7], 3 * cap, 3)
    nets, live = {}, {}
    for i, which in enumerate(("mapping", "atlas")):
        off = (C.c_int64 * OFFSETS)()
        N.check(lib.b200_atlas_tc_image_offsets_for(C.byref(cfg), C.byref(tr.map_desc), N.ptr(ws), i, off), "offsets")
        dims = NETS[which][0]
        net = Net(dims, tr.params[tr.net_slice(which)])
        tiles = map_tiles if i == 0 else atl_tiles
        nets[which] = (net, Images(ws, off, net, tiles), off)
        live[which] = len(tiles)
    worst = Worst()
    gemms = []
    for which, groups in (("mapping", ng), ("atlas", 3)):
        gemms += [(a, b, groups) for _, a, b in wgrad_gemms(nets[which][0])]
    n_split = unit_splits(gemms, wg_units)
    first = 0
    for i, which in enumerate(("mapping", "atlas")):
        net, im, off = nets[which]
        tiles = map_tiles if i == 0 else atl_tiles
        r = rows_of(tiles)
        if i == 0:
            inp, y, dy = x_map[r], uv[r], d_uv[r]
        else:
            inp, y, dy = uv[r] * 0.5 + 0.5, y_atl[r], d_y[r]
        s_g = grad_scale(int(ws[off[GMAX]:off[GMAX] + 8].view(torch.int32)[1 - i]))
        check_weight_images(im, net, worst)
        check_forward(im, net, inp, y, worst)
        check_backward(im, net, y, dy, s_g, worst)
        k = len(wgrad_gemms(net))
        check_weight_gradients(im, net, tr.grads[tr.net_slice(which)], s_g, live[which], n_split[first:first + k], worst)
        first += k
    worst.report(f"fused step, {'with' if with_global else 'without'} the global rigidity term, "
                 f"{live['mapping']} + {live['atlas']} live tiles")
