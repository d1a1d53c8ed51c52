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
    s_g is recomputed from the gmax word the call used with the rule of `grad_scales`.  No hi term of an activation,
    encoding or dZ image may be +-65504: there the saturating split has lost its 22 bits.

Stand-alone calls: the `IMLP` call for the six networks with tensor-core kernels at the row counts of
test_wgrad_gpu.py and test_bwd_reductions_gpu.py (1, 127, 129, one tile per cluster of two SMs less / more one tile,
3 * 132 * 128 - 50); the atlas input gradient overwrites d_in there.  Bias gradients and the plain mapping's dW0 are
test_bwd_reductions_gpu.py's.

The fused stage-1 trip (b200_atlas_loss_grad_for at B200_PREC_TC): the mapping on 9 * cap planned rows in nine or
seven groups (with / without the global rigidity term; groups 5 / 6 compacted to counters[5] / [6] rows), the atlas on
3 groups of counters[0] rows, one work list for both networks.  The trip workspace is filled with 0xFF first; the
live tiles come from `live_tiles`, a host mirror of TileIter on the device counters, which must equal a host count.
Per network, on the live tiles: (a) to (d) above; every dead tile's output rows, activation / dZ / encoding images
and flag words still hold the fill (in the seven-group regime groups 7 and 8 are dead entirely), every live output
row is finite and every x_map row of a live tile past its group's count is zero; the atlas's gmax word is max |d_y| and the mapping's is at least max |d_uv|.  d_uv of groups 0-2 is
the loss head's gradient plus 0.5 times the atlas input gradient: the head is test_stage1_heads_gpu.atlas_head in
float64 on the device's own uv / y / targets within its envelope, the addend comes from the atlas's own dZ and
encoding images (`check_input_gradient` with a base).  Cases, each asserting the TileIter edge it covers:
  fullsize        80 x 432 x 768, B = 10 000, with and without the global term (test_fused_step_layers)
  shard           the same, 2 and 8 ways, rank 0 and the last rank: most tiles dead, tile counts differ per rank
  small shard     rank 0 of 2 on a 32 x 48 x 4 video, 1 / 127 / 128 / 129 resident rows x no forward-flow row, all
                  rows forward-valid, forward rows a multiple of 128
  small whole     B = 1 / 127 / 128 / 129: sample_kernel<true> writes its own padding rows
  empty shard     zero tiles: every row keeps the fill, the gradients are zero, losses[6:8] the whole batch's counts
  cached          eager trips, then graph replays of both regimes in turn on counts that move in opposite
                  directions, before and after a pre-training sweep on the shared workspace
  pe mapping      use_positional_encoding_mapping1 with 1 and 10 frequencies, whole video and rank 0 of 2
The pre-training trip (b200_pretrain_loss_grad_for): B = 1 / 127 / 128 / 129 / 10 000, plain and PE-10 mappings, on a
0xFF workspace: counters[0] = B, the mapping's layers on one group with a mapping-only work list, its other groups
dead, every atlas image and buffer untouched and the atlas block of the gradients left as it was.
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
from tc_images_common import (ATOM, B_SMALL, DEV, FRAME, GMAX, OFFSETS, SMALL, TM, Images, Net, Worst, _need_tc,
                              check_backward, check_forward, check_input_gradient, check_weight_gradients,
                              check_weight_images, desc_dims, flow_counts, grad_scale, host_counts, live_tiles,
                              run_trip, small_batch, small_data, tiles_of, unit_splits, wg_units,
                              wgrad_gemms)  # noqa: F401  (wg_units: a fixture)
from test_stage1_heads_gpu import G_BWD, G_FWD, _atlas_views, atlas_head

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
    dims, xs, xo = NETS[which]
    g = torch.Generator().manual_seed(_seed(f"{which}/{rows}"))
    net = Net(dims, None)
    net.flat = _init_flat(net, g)
    x = (torch.rand(rows, net.in_dim, generator=g) * xs + xo).to(DEV)
    dy = torch.randn(rows, net.out, generator=g).to(DEV)
    check_imlp(net, x, dy, wg_units, f"{which} rows {rows}")


def check_imlp(net, x, dy, wg_units, label):
    """Runs the stand-alone IMLP call of `net` on x and dy on a 0xFF workspace and applies checks (a) to (d).
    Returns the decoded images and what the call wrote: dict(im, s_g, word, grads, d_in)."""
    lib = N.lib()
    rows = x.shape[0]
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
    worst.report(label)
    return dict(im=im, s_g=s_g, word=word, grads=grads, d_in=d_in)


# ---------------------------------------------------------------------------------------------------------------
# the fused stage-1 trip (b200_atlas_loss_grad_for) and the pre-training trip (b200_pretrain_loss_grad_for)
# ---------------------------------------------------------------------------------------------------------------
FULL = dict(T=80, H=432, W=768, B=10000)


def _live_mask(n_tiles, tiles):
    live = torch.zeros(n_tiles, dtype=torch.bool, device=DEV)
    live[torch.as_tensor(tiles, dtype=torch.long, device=DEV)] = True
    return live


def _rows_of(tiles):
    return (torch.as_tensor(tiles, dtype=torch.long, device=DEV)[:, None] * TM + torch.arange(TM, device=DEV)).flatten()


def _holds_fill(ws, begin, end):
    return bool((ws[begin:end] == 0xFF).all())


def _f32(word):
    return float(np.int32(word).view(np.float32))


def check_dead_tiles(ws, off, net, y_all, live, label):
    """Every dead tile's output rows, activation, dZ, encoding and output-dZ images and flag words still hold the
    0xFF fill; every output row of a live tile is finite."""
    o = [int(v) for v in off]
    n_tiles = live.numel()
    y_t = y_all.reshape(n_tiles, -1)
    assert bool((y_t.view(torch.int32)[~live] == -1).all()), f"{label}: a dead tile's output was written"
    assert bool(torch.isfinite(y_t[live]).all()), f"{label}: an output row of a live tile is not finite"
    for what, base in (("activation", o[3]), ("dZ", o[4])):
        img = ws[base:base + (net.L - 1) * o[8]].view(net.L - 1, 2, n_tiles, -1)
        assert bool((img[:, :, ~live] == 0xFF).all()), f"{label}: a dead tile's {what} image was written"
    for what, base in (("encoding", o[5]), ("output dZ", o[6])):
        for t in range(2 if base >= 0 else 0):
            img = ws[base + t * o[10]:base + t * o[10] + n_tiles * ATOM].view(n_tiles, -1)
            assert bool((img[~live] == 0xFF).all()), f"{label}: a dead tile's {what} image was written"
    flags = ws[o[7]:o[7] + (net.L - 1) * o[11] * 32].view(net.L - 1, n_tiles, -1)
    assert bool((flags[:, ~live] == 0xFF).all()), f"{label}: a dead tile's flag words were written"


def head_d_uv(tr, cfg, ws, ng, label):
    """The loss head's d_uv of groups 0-2 in float64 (test_stage1_heads_gpu.atlas_head, with its envelope) from the
    device's own uv, y and targets: value and bound as [3 cap, 2] tensors, zero past counters[0]; an undecidable
    sample gets an infinite bound (only finiteness is checked), and the cases here must have none."""
    v = _atlas_views(tr, cfg, ws)
    cap, cnt = v["cap"], v["counters"]
    n = int(cnt[0])
    val, bnd = np.zeros((3, cap, 2)), np.zeros((3, cap, 2))
    if n:
        tg = v["targets"][:n]
        pf, pb = tg[:, 9].astype(np.int64) - 1, tg[:, 10].astype(np.int64) - 1
        s = np.arange(n)
        rows = [np.maximum(pf, 0) if g == G_FWD else (np.maximum(pb, 0) if g == G_BWD else s) for g in range(9)]
        uv = np.stack([np.where((g < ng) & ((g != G_FWD) | (pf >= 0)) & ((g != G_BWD) | (pb >= 0)),
                                v["uv"][g, rows[g]].T, 0).T for g in range(9)])
        duv, _, _, und = atlas_head(uv, v["y"][:, :n], tg, pf >= 0, pb >= 0, cfg, max(tr.video.H, tr.video.W),
                                    cfg.batch, int(cnt[1]), int(cnt[2]), ng)
        assert not und.any(), f"{label}: {int(und.sum())} samples with an undecidable loss-head branch"
        for g in range(3):
            for c in range(2):
                val[g, :n, c] = np.where(und, 0.0, duv[g][c].v)
                bnd[g, :n, c] = np.where(und, np.inf, duv[g][c].bound())
    as_dev = lambda a: torch.from_numpy(a.reshape(3 * cap, 2)).to(DEV)
    return as_dev(val), as_dev(bnd)


def check_atlas_trip(tr, with_global, want_counts, wg_units, label, keep=None):
    """Checks (a) to (d) of both networks of the trip `tr` just ran on a 0xFF workspace, the tiles each launch
    visited, the counters, the gmax words and the summed d_uv of groups 0-2.  Returns the counters; appends
    (network name, Images, s_g, gmax word) per network to the list `keep` when one is given."""
    lib = N.lib()
    cfg = tr._config(with_global)
    ws = tr._workspace()
    ng = 9 if with_global else 7
    cap = -(-int(cfg.batch) // TM) * TM
    wo = (C.c_int64 * 8)()
    N.check(lib.b200_atlas_workspace_offsets_for(C.byref(cfg), C.byref(tr.map_desc), N.ptr(ws), wo), "offsets")
    cnt = [int(v) for v in ws[wo[0]:wo[0] + 32].view(torch.int32).cpu()]
    assert (cnt[0], cnt[5], cnt[6]) == tuple(want_counts), (label, cnt[:7], want_counts)
    f32 = lambda o, n, w: ws[o:o + 4 * n * w].view(torch.float32).view(n, w)
    x_map, d_uv, uv = f32(wo[2], 9 * cap, 4), f32(wo[4], 9 * cap, 2), f32(wo[6], 9 * cap, 2)
    d_y, y_atl = f32(wo[5], 3 * cap, 3), f32(wo[7], 3 * cap, 3)
    assert bool((d_uv[ng * cap:].view(torch.int32) == -1).all()), f"{label}: d_uv of a group past {ng - 1} written"
    # the rows of a live tile past its group's count are zero in x_map (a NaN there can vanish in a plain mapping's
    # first ReLU, so finite outputs do not show it)
    for g in range(ng):
        lim = cnt[5] if g == G_FWD else (cnt[6] if g == G_BWD else cnt[0])
        pad = x_map[g * cap + lim:g * cap + min(cap, tiles_of(lim) * TM)]
        assert bool((pad == 0).all()), f"{label}: x_map group {g} rows past {lim} in a live tile are not zero"
    head, head_bound = head_d_uv(tr, cfg, ws, ng, label)
    nets, gemms = [], []
    for i, which in enumerate(("mapping", "atlas")):
        off = (C.c_int64 * OFFSETS)()
        N.check(lib.b200_atlas_tc_image_offsets_for(C.byref(cfg), C.byref(tr.map_desc), N.ptr(ws), i, off), "offsets")
        assert off[11] == (9 if i == 0 else 3) * cap
        net = Net(desc_dims(tr.descs[which]), tr.params[tr.net_slice(which)])
        groups = ng if i == 0 else 3
        tiles = live_tiles(cap, groups, cnt, G_FWD, G_BWD) if i == 0 else live_tiles(cap, 3, cnt, -1, -1)
        nets.append((which, net, off, tiles))
        gemms += [(a, b, groups) for _, a, b in wgrad_gemms(net)]
    n_split = unit_splits(gemms, wg_units)
    first, worst_all, summed = 0, 0.0, 0.0
    for i, (which, net, off, tiles) in enumerate(nets):
        check_dead_tiles(ws, off, net, uv if i == 0 else y_atl, _live_mask(int(off[11]) // TM, tiles),
                         f"{label}, {which}")
        r = _rows_of(tiles)
        if i == 0:
            inp, y, dy = x_map[r], uv[r], d_uv[r]
            word = cnt[4]
            mx = float(d_uv[:ng * cap].abs().max())
            assert _f32(word) >= mx, f"{label}: the mapping's gmax word {_f32(word)} is below max |d_uv| {mx}"
        else:
            inp, y, dy = uv[r] * 0.5 + 0.5, y_atl[r], d_y[r]
            word = cnt[3]
            assert word == int(d_y.abs().max().view(torch.int32)), f"{label}: the atlas's gmax word is not max |d_y|"
        s_g = grad_scale(word)
        im = Images(ws, off, net, tiles)
        worst = Worst()
        check_weight_images(im, net, worst)
        check_forward(im, net, inp, y, worst)
        check_backward(im, net, y, dy, s_g, worst)
        if i == 1:
            check_input_gradient(im, net, s_g, d_uv[r], worst, base=(head[r], head_bound[r]))
            summed = worst.r["d_in + head"]
        k = len(wgrad_gemms(net))
        check_weight_gradients(im, net, tr.grads[tr.net_slice(which)], s_g, len(tiles), n_split[first:first + k], worst)
        first += k
        if keep is not None:
            keep.append((which, im, s_g, word))
        worst_all = max(worst_all, worst.report(f"{label}, {which}: {len(tiles)} of {int(off[11]) // TM} tiles live"))
    print(f"{label}: largest error / bound over both networks {worst_all:.3g}, summed d_uv of groups 0-2 {summed:.3g}")
    return cnt


def _trainer(data, B, t0=0, t1=None, pe=0, state=None):
    """An AtlasTrainer on frames [t0, t1) of `data` at B_PREC_TC: the given (mapping, atlas) state dicts, or the
    reference initialisation."""
    conf = {"samples_batch": B}
    if pe:
        conf.update(use_positional_encoding_mapping1=True, number_of_positional_encoding_mapping1=pe)
    tr = A.AtlasTrainer(A.DeviceVideo.from_reference_layout(data, DEV, t0, t1), conf, precision=N.PREC_TC, device=DEV)
    if state is None:
        torch.manual_seed(11)
        tr.init_like_reference()
    else:
        tr.load_state(*state)
    return tr


# ---------------------------------------------------------------------------------------------------------------
# benchmark geometry
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def fullsize(golden_dir):
    """The benchmark's video, an index batch and the golden parameters."""
    _need_tc()
    T, H, W, B = FULL["T"], FULL["H"], FULL["W"], FULL["B"]
    data = synth.throughput_set(H, W, T, seed=0)
    z = np.load(os.path.join(golden_dir, "params_seed1234.npz"))
    state = (O.state_dict_of([torch.from_numpy(z[f"map{i}"]) for i in range(12)]),
             O.state_dict_of([torch.from_numpy(z[f"atl{i}"]) for i in range(16)]))
    inds = torch.randint(H * W * T, (B,), generator=torch.Generator().manual_seed(1))
    return data, inds, state


@pytest.mark.parametrize("with_global", [True, False])
def test_fused_step_layers(fullsize, with_global, wg_units):
    """The whole video at the benchmark shape: every tile of the ordinary groups live, the compacted flow groups
    fewer and not tile-aligned."""
    data, inds, state = fullsize
    T, H, W, B = FULL["T"], FULL["H"], FULL["W"], FULL["B"]
    want = host_counts(inds, data, 0, T, H, W)
    n, nf, nb = want
    assert n == B and tiles_of(nf) < tiles_of(n) and tiles_of(nb) < tiles_of(n) and (nf % TM or nb % TM), want
    tr = _trainer(data, B, state=state)
    tr.indices.copy_(inds)
    run_trip(tr, with_global)
    check_atlas_trip(tr, with_global, want, wg_units,
                     f"fused step, {'with' if with_global else 'without'} the global rigidity term")


@pytest.mark.parametrize("world,rank", [(2, 0), (2, 1), (8, 0), (8, 7)])
def test_fused_step_shard_layers(fullsize, world, rank, wg_units):
    """One frame shard (sample_kernel<false>: claimed slots, the x_map memset of every group): counters[0] far below
    cap, so most tiles of every group are dead; rank 0's and the last rank's tile counts differ."""
    data, inds, state = fullsize
    T, H, W, B = FULL["T"], FULL["H"], FULL["W"], FULL["B"]
    per_rank = []
    for r in (0, world - 1):
        n, nf, nb = host_counts(inds, data, *A.frame_range(r, world, T), H, W)
        per_rank.append((tiles_of(n), tiles_of(nf), tiles_of(nb)))
        assert tiles_of(nf) < tiles_of(n) < tiles_of(B) and tiles_of(nb) < tiles_of(n), (r, n, nf, nb)
    assert per_rank[0] != per_rank[1], per_rank
    t0, t1 = A.frame_range(rank, world, T)
    tr = _trainer(data, B, t0, t1, state=state)
    tr.indices.copy_(inds)
    run_trip(tr, True)
    check_atlas_trip(tr, True, host_counts(inds, data, t0, t1, H, W), wg_units, f"{world}-way shard, rank {rank}")


# ---------------------------------------------------------------------------------------------------------------
# tile edges on a small video
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("regime", ["no_fwd", "all_fwd", "fwd_whole_tiles"])
@pytest.mark.parametrize("n_local", [1, 127, 128, 129])
def test_small_shard_layers(n_local, regime, wg_units):
    """Rank 0 of 2 on hand-built batches: 1 / 127 / 128 / 129 resident rows and a compacted group with no tile, one
    equal to the ordinary groups, or a full last tile beside a partial one."""
    _need_tc()
    n_f, n_b = flow_counts(n_local, regime)
    data, _ = small_data()
    T, H, W = SMALL["T"], SMALL["H"], SMALL["W"]
    t0, t1 = A.frame_range(0, 2, T)
    assert t0 <= FRAME < t1
    inds = small_batch(n_local, n_f, n_b, seed=n_local)
    want = host_counts(inds, data, t0, t1, H, W)
    assert want == (n_local, n_f, n_b), want
    if regime == "no_fwd":
        assert n_f == 0 and n_b > 0                                 # a compacted group with no tile at all
    elif regime == "all_fwd":
        assert n_f == n_local                                       # compacted group = ordinary group
    else:
        assert n_f % TM == 0 and n_b % TM != 0                      # a full last tile beside a partial one
    tr = _trainer(data, B_SMALL, t0, t1)
    tr.indices.copy_(inds)
    run_trip(tr, True)
    check_atlas_trip(tr, True, want, wg_units, f"small shard, n_local {n_local}, {regime} ({n_f} / {n_b} flow rows)")


@pytest.mark.parametrize("B", [1, 127, 128, 129])
def test_small_whole_video_layers(B, wg_units):
    """The whole video (sample_kernel<true>, which writes its own padding rows: only the flow-match groups are
    cleared first): every tile of the ordinary groups live, the last one holding B % 128 samples (none padded at
    128)."""
    _need_tc()
    data, _ = small_data()
    T, H, W = SMALL["T"], SMALL["H"], SMALL["W"]
    inds = torch.randint(H * W * T, (B,), generator=torch.Generator().manual_seed(B))
    want = host_counts(inds, data, 0, T, H, W)
    assert want[0] == B and tiles_of(B) == 1 + (B > TM)
    tr = _trainer(data, B)
    tr.indices.copy_(inds)
    run_trip(tr, True)
    check_atlas_trip(tr, True, want, wg_units, f"small whole video, B {B} ({want[1]} / {want[2]} flow rows)")


def test_empty_shard_layers(wg_units):
    """Rank 1 of 2 holds no sample of the batch: zero tiles run (every output row and image keeps the fill), the
    gradients are exactly zero and the loss vector still carries the whole batch's flow counts."""
    _need_tc()
    data, _ = small_data()
    T, H, W = SMALL["T"], SMALL["H"], SMALL["W"]
    inds = FRAME * H * W + torch.randint(H * W, (B_SMALL,), generator=torch.Generator().manual_seed(9))
    t0, t1 = A.frame_range(1, 2, T)
    assert not t0 <= FRAME < t1
    tr = _trainer(data, B_SMALL, t0, t1)
    tr.indices.copy_(inds)
    run_trip(tr, True)
    cnt = check_atlas_trip(tr, True, (0, 0, 0), wg_units, "empty shard")
    _, n_f, n_b = host_counts(inds, data, 0, T, H, W)
    assert (cnt[1], cnt[2]) == (n_f, n_b) and n_f > 0 and n_b > 0
    assert tr.losses[6:8].tolist() == [n_f, n_b]
    assert torch.count_nonzero(tr.grads) == 0


def test_cached_work_lists_layers(wg_units):
    """One trainer, rank 0 of 2: an eager trip per regime (they cache the job tables and work lists, one entry per
    regime, keyed on the row geometry and not on the counts), then graph replays of both regimes in turn on batches
    whose resident and forward-flow tile counts move in opposite directions, before and after a pre-training sweep
    on the shared workspace (its own cache entry, on a plan carved at cap = 10 112)."""
    _need_tc()
    data, _ = small_data()
    T, H, W = SMALL["T"], SMALL["H"], SMALL["W"]
    t0, t1 = A.frame_range(0, 2, T)
    tr = _trainer(data, B_SMALL, t0, t1)
    first = (140, 130, 20)
    trips = [(True, (300, 100, 250)), (False, (129, 129, 1)), (True, (385, 0, 384)), "pretrain",
             (False, (127, 127, 64)), (True, (300, 0, 250))]
    counts = [first] + [c for _, c in (t for t in trips if t != "pretrain")]
    for a, b in zip(counts, counts[1:]):
        assert (tiles_of(b[0]) - tiles_of(a[0])) * (tiles_of(b[1]) - tiles_of(a[1])) < 0, (a, b)
    tr.indices.copy_(small_batch(*first, seed=1))
    graphs = {}
    for wg in (True, False):
        run_trip(tr, wg)
        check_atlas_trip(tr, wg, first, wg_units, f"cached work lists, eager trip {'with' if wg else 'without'}")
        graphs[wg] = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graphs[wg]):
            tr.loss_grad(wg)
    for k, trip in enumerate(trips):
        if trip == "pretrain":
            tr.pretrain(T, H, W, 1, generator=torch.Generator().manual_seed(3))
            torch.cuda.synchronize()
            continue
        wg, c = trip
        tr.indices.copy_(small_batch(*c, seed=10 + k))
        run_trip(tr, wg, replay=graphs[wg])
        check_atlas_trip(tr, wg, c, wg_units, f"cached work lists, replay {k} {'with' if wg else 'without'} {c}")


@pytest.mark.parametrize("world", [1, 2])
@pytest.mark.parametrize("pe", [1, 10])
def test_pe_mapping_layers(pe, world, wg_units):
    """use_positional_encoding_mapping1 with 1 and 10 frequencies (6 and 60 encoding columns): the mapping on the
    position-encoded kernels (network code 4), whole video and rank 0 of 2."""
    _need_tc()
    data, _ = small_data()
    T, H, W = SMALL["T"], SMALL["H"], SMALL["W"]
    t0, t1 = A.frame_range(0, world, T)
    tr = _trainer(data, B_SMALL, t0, t1, pe=pe)
    assert N.lib().b200_mlp_tc_architecture(C.byref(tr.map_desc)) == 4
    inds = torch.randint(H * W * T, (B_SMALL,), generator=torch.Generator().manual_seed(4))
    want = host_counts(inds, data, t0, t1, H, W)
    assert 0 < want[0] <= B_SMALL and (want[0] == B_SMALL) == (world == 1) and 0 < want[1] < want[0]
    tr.indices.copy_(inds)
    run_trip(tr, True)
    check_atlas_trip(tr, True, want, wg_units, f"PE-{pe} mapping, {'whole video' if world == 1 else 'rank 0 of 2'}")


# ---------------------------------------------------------------------------------------------------------------
# the pre-training trip
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [1, 127, 128, 129, 10000])
@pytest.mark.parametrize("pe", [0, 10])
def test_pretrain_trip_layers(pe, B, wg_units):
    """b200_pretrain_loss_grad_for on a 0xFF workspace: the mapping alone on one group of B rows (its own work list);
    the other mapping groups, every atlas image and buffer, and the atlas block of the gradients stay untouched."""
    _need_tc()
    data, _ = small_data()
    tr = _trainer(data, B_SMALL, pe=pe)
    check_pretrain_trip(tr, B, wg_units, f"pre-training trip, {'plain' if pe == 0 else f'PE-{pe}'} mapping, B {B}")


def check_pretrain_trip(tr, B, wg_units, label):
    """One pre-training trip of B random pixels of the benchmark geometry on the mapping of `tr`, checked as
    test_pretrain_trip_layers states.  Returns the mapping's Images, s_g and gmax word."""
    lib = N.lib()
    H, W, T, f = FULL["H"], FULL["W"], FULL["T"], 37
    g = torch.Generator().manual_seed(B)
    ys, xs = torch.randint(H, (B,), generator=g).to(DEV), torch.randint(W, (B,), generator=g).to(DEV)
    cfg = tr._config(False)
    cfg.batch = B
    ws = torch.full((int(lib.b200_atlas_workspace_bytes_for(C.byref(cfg), C.byref(tr.map_desc))),), 0xFF,
                    dtype=torch.uint8, device=DEV)
    atl = tr.grads[tr.net_slice("atlas")]
    atl.fill_(float("nan"))
    nan_bits = int(atl[:1].view(torch.int32)[0])
    N.check(lib.b200_pretrain_loss_grad_for(C.byref(cfg), C.byref(tr.map_desc), max(H, W), T, f, N.ptr(ys), N.ptr(xs),
                                            N.ptr(tr.params), N.ptr(tr.grads), N.ptr(tr.losses), N.ptr(ws), ws.numel(),
                                            N.current_stream()), "b200_pretrain_loss_grad_for")
    torch.cuda.synchronize()
    assert bool((atl.view(torch.int32) == nan_bits).all()), f"{label}: the atlas gradients were written"
    cap = tiles_of(B) * TM
    wo = (C.c_int64 * 8)()
    N.check(lib.b200_atlas_workspace_offsets_for(C.byref(cfg), C.byref(tr.map_desc), N.ptr(ws), wo), "offsets")
    cnt = [int(v) for v in ws[wo[0]:wo[0] + 32].view(torch.int32).cpu()]
    assert cnt[0] == B and cnt[3] == 0, cnt[:7]
    f32 = lambda o, n, w: ws[o:o + 4 * n * w].view(torch.float32).view(n, w)
    x_map, d_uv, uv = f32(wo[2], 9 * cap, 4), f32(wo[4], 9 * cap, 2), f32(wo[6], 9 * cap, 2)
    assert _holds_fill(ws, wo[4] + 8 * cap, wo[4] + 8 * 9 * cap), f"{label}: d_uv past group 0 written"
    # the atlas: every image, its output and its output gradient keep the fill
    off_a = (C.c_int64 * OFFSETS)()
    N.check(lib.b200_atlas_tc_image_offsets_for(C.byref(cfg), C.byref(tr.map_desc), N.ptr(ws), 1, off_a), "offsets")
    begin = min(int(off_a[k]) for k in range(8) if off_a[k] >= 0)
    assert _holds_fill(ws, begin, off_a[7] + (8 - 1) * off_a[11] * 32), f"{label}: an atlas image was written"
    assert _holds_fill(ws, wo[5], wo[5] + 4 * 3 * cap * 3) and _holds_fill(ws, wo[7], wo[7] + 4 * 3 * cap * 3), \
        f"{label}: the atlas's output or its gradient was written"
    # the mapping: one group of tiles_of(B) tiles
    off = (C.c_int64 * OFFSETS)()
    N.check(lib.b200_atlas_tc_image_offsets_for(C.byref(cfg), C.byref(tr.map_desc), N.ptr(ws), 0, off), "offsets")
    assert off[11] == 9 * cap
    net = Net(desc_dims(tr.map_desc), tr.params[tr.net_slice("mapping")])
    tiles = live_tiles(cap, 1, cnt, -1, -1)
    assert len(tiles) == tiles_of(B)
    check_dead_tiles(ws, off, net, uv, _live_mask(9 * cap // TM, tiles), label)
    word = cnt[4]
    assert word == int(d_uv[:cap].abs().max().view(torch.int32)), f"{label}: the gmax word is not max |d_uv|"
    s_g = grad_scale(word)
    r = _rows_of(tiles)
    im = Images(ws, off, net, tiles)
    worst = Worst()
    check_weight_images(im, net, worst)
    check_forward(im, net, x_map[r], uv[r], worst)
    check_backward(im, net, uv[r], d_uv[r], s_g, worst)
    n_split = unit_splits([(a, b, 1) for _, a, b in wgrad_gemms(net)], wg_units)
    check_weight_gradients(im, net, tr.grads[tr.net_slice("mapping")], s_g, len(tiles), n_split, worst)
    worst.report(f"{label}: {len(tiles)} of {9 * cap // TM} tiles live")
    return im, s_g, word
