"""The segmentation trip's tensor-core launches (b200_seg_loss_grad at B200_PREC_TC: mapping1, mapping2, alpha and
atlas, each a counted stand-alone call of csrc/mlp_tc.cu on a group-major batch) one layer at a time against float64
references built from the operands the kernels themselves read, with the checks and the bound of
test_tc_layers_gpu.py (tc_images_common.py, c = 4).

Before each checked trip the whole trip workspace is filled with 0xFF (NaN in every float and fp16 pair); the
networks' job tables live outside it.  For every network b200_seg_tc_image_offsets locates the images in the
network's slice, and the live tiles come from `live_tiles`, a host mirror of TileIter applied to the device counters
(counters[0] rows in every group, counters[5] / [6] in the compacted groups: 5 / 6 of the mappings' 9 or 7 groups,
3 / 4 of alpha's 5; the atlas's 6 groups are not compacted).  Checked per network, on the live tiles:
  (a) the weight items and forward constants, bit for bit;
  (b) every activation image, flag word, the encoding image and the output;
  (c) every dZ image and the output-layer dZ, with s_g recomputed from the gmax word (asserted to be max |dy|);
      the atlas input gradient d_xat, which the counted call overwrites;
  (d) every dW of the call's own work list (`unit_splits` over this network's GEMMs and groups).
and, so that a launch that evaluates tiles it should not cannot pass (extra rows have zero dy and change no value):
every row of a dead tile in the network's output (and in d_xat), and in every activation image, still holds the
fill, and every row of a live tile is finite.  The counters must equal a host count from the index batch, the shard
and the flow masks.

Cases (each asserts on the host the TileIter edge it is there for):
  fullsize      80 x 432 x 768, B = 10 000, after one pre-training sweep of both mappings, with and without the
                global rigidity term: compacted groups with fewer live tiles than the others, not tile-aligned
  shard         the same geometry split 2 and 8 ways, rank 0 and the last rank: far fewer resident rows than cap,
                so most tiles of every group are dead, and the two ranks' tile counts differ
  small         hand-built batches on a 32 x 48 x 4 video, rank 0 of a 2-way split, n_local in {1, 127, 128, 129}:
                no forward-flow row while backward rows exist (a compacted group with zero tiles), every resident
                row forward-valid (compacted group = ordinary group), forward rows a multiple of 128 while the
                backward rows are not (a full last tile next to a partial one)
  empty shard   a rank with no resident sample: zero tiles run, every output row holds the fill, gradients zero
  cached        two trips on one SegTrainer whose counts move in opposite directions (more resident rows, fewer
                forward-flow rows); the second trip is a CUDA-graph replay on the work lists the first one cached
  pe mappings   use_positional_encoding_mapping1/2: both mappings on the position-encoded kernels (network code 4)
Each case prints its largest ratio of error to bound per network (`pytest -s`).

test_seg_render_matches_training_forwards: b200_seg_render's inference forwards (no images stored) are bit-identical
to training-mode forwards at the render's row counts, and its composite is restated in float32 bit for bit.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from b200 import _native as N
from b200 import atlas as A
from b200 import seg as SG
from b200 import synth
from tc_images_common import (B_SMALL, DEV, FRAME, GMAX, OFFSETS, SMALL, TM, Images, Net, Worst, _need_tc,
                              check_backward, check_forward, check_input_gradient, check_weight_gradients,
                              check_weight_images, desc_dims, flow_counts, grad_scale, host_counts, live_tiles,
                              run_trip, small_batch, small_data, tiles_of, unit_splits, wg_units,
                              wgrad_gemms)  # noqa: F401  (wg_units: a fixture)

pytestmark = pytest.mark.gpu

# per network: input buffer, output buffer, output-gradient buffer (indices of b200_seg_workspace_offsets), input
# columns, compacted groups
ROLES = {"mapping1": (3, 6, 10, 3, 5, 6), "mapping2": (3, 7, 11, 3, 5, 6), "alpha": (4, 8, 12, 3, 3, 4),
         "atlas": (5, 9, 13, 2, -1, -1)}
D_XAT = 14
FULL = dict(T=80, H=432, W=768, B=10000)


def check_trip(tr, it, want_counts, wg_units, label):
    """Checks (a) to (d), the visited tiles and the counters of the trip `tr` just ran; returns the counters."""
    lib = N.lib()
    cfg = tr._config(it)
    ws = tr._workspace()
    wo = (C.c_int64 * N.SEG_OFFSET_FLOATS)()
    N.check(lib.b200_seg_workspace_offsets(C.byref(cfg), N.ptr(ws), wo), "trip offsets")
    cap = -(-int(cfg.batch) // TM) * TM
    cnt = [int(v) for v in ws[wo[0]:wo[0] + 32].view(torch.int32).cpu()]
    assert (cnt[0], cnt[5], cnt[6]) == tuple(want_counts), (label, cnt[:7], want_counts)
    buf = lambda i, rows, w: ws[wo[i]:wo[i] + 4 * rows * w].view(torch.float32).view(rows, w)
    worst_all = 0.0
    for k, which in enumerate(SG.NETS):
        assert lib.b200_mlp_tc_architecture(C.byref(tr.descs[which])) > 0, which
        off = (C.c_int64 * OFFSETS)()
        N.check(lib.b200_seg_tc_image_offsets(C.byref(cfg), N.ptr(ws), k, off), f"{which} image offsets")
        rows = int(off[11])
        groups = rows // cap
        assert groups == {0: 9 if cfg.with_global else 7, 1: 9 if cfg.with_global else 7, 2: 5, 3: 6}[k]
        i_in, i_out, i_dy, cols, g_fwd, g_bwd = ROLES[which]
        net = Net(desc_dims(tr.descs[which]), tr.params[tr.net_slice(which)])
        tiles = live_tiles(cap, groups, cnt, g_fwd, g_bwd)
        n_tiles = rows // TM
        live = torch.zeros(n_tiles, dtype=torch.bool, device=DEV)
        live[torch.as_tensor(tiles, dtype=torch.long, device=DEV)] = True
        # exactly the live tiles: dead rows of the output and of every activation image still hold the fill
        y_all = buf(i_out, rows, net.out)
        y_bits = y_all.view(torch.int32).view(n_tiles, TM * net.out)
        assert bool((y_bits[~live] == -1).all()), f"{label} {which}: a dead tile's output was written"
        assert bool(torch.isfinite(y_all.view(n_tiles, TM * net.out)[live]).all()), f"{label} {which}: live output"
        act = ws[off[3]:off[3] + (net.L - 1) * off[8]].view(torch.int16).view(net.L - 1, 2, n_tiles, -1)
        assert bool((act[:, :, ~live] == -1).all()), f"{label} {which}: a dead tile's activation image was written"
        if which == "atlas":
            d_x = buf(D_XAT, rows, 2)
            assert bool((d_x.view(torch.int32).view(n_tiles, -1)[~live] == -1).all()), f"{label}: dead d_xat rows"
        dy_all = buf(i_dy, rows, net.out)
        word = int(ws[off[GMAX]:off[GMAX] + 8].view(torch.int32)[1 if net.out == 2 else 0])
        assert word == int(dy_all.abs().max().view(torch.int32)), f"{label} {which}: the gmax word is not max |dy|"
        s_g = grad_scale(word)
        im = Images(ws, off, net, tiles)
        r = (torch.as_tensor(tiles, dtype=torch.long, device=DEV)[:, None] * TM
             + torch.arange(TM, device=DEV)).flatten()
        inp, y, dy = buf(i_in, rows, cols)[r], y_all[r], dy_all[r]
        worst = Worst()
        check_weight_images(im, net, worst)
        check_forward(im, net, inp, y, worst)
        check_backward(im, net, y, dy, s_g, worst)
        if which == "atlas":
            check_input_gradient(im, net, s_g, d_x[r], worst)
        gemms = wgrad_gemms(net)
        n_split = unit_splits([(a, b, groups) for _, a, b in gemms], wg_units)
        check_weight_gradients(im, net, tr.grads[tr.net_slice(which)], s_g, len(tiles), n_split, worst)
        worst.report(f"{label}, {which}: {len(tiles)} of {n_tiles} tiles live")
        worst_all = max(worst_all, max(worst.r.values()))
    print(f"{label}: largest error / bound over the four networks {worst_all:.3g}")
    return cnt


# ---------------------------------------------------------------------------------------------------------------
# benchmark geometry
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def fullsize():
    """The data, matte, index batch and parameters (reference init, one pre-training sweep of both mappings) of
    test_seg_fullsize_gpu.py."""
    _need_tc()
    T, H, W, B = FULL["T"], FULL["H"], FULL["W"], FULL["B"]
    data = synth.throughput_set(H, W, T, seed=0)
    masks = (torch.rand(H, W, T, generator=torch.Generator().manual_seed(2)) < 0.4).float()
    tr = SG.SegTrainer(A.DeviceVideo.from_reference_layout(data, DEV), SG.pack_mask_frames(masks, DEV), None,
                       precision=N.PREC_TC, device=DEV)
    torch.manual_seed(11)
    tr.init_like_reference()
    for which in ("mapping1", "mapping2"):
        tr.pretrain(which, T, H, W, 1)
    inds = torch.randint(H * W * T, (B,), generator=torch.Generator().manual_seed(3))
    params = tr.params.detach().clone()
    del tr
    torch.cuda.empty_cache()
    return data, masks, inds, params


def _fullsize_trainer(fullsize, t0, t1):
    data, masks, inds, params = fullsize
    tr = SG.SegTrainer(A.DeviceVideo.from_reference_layout(data, DEV, t0, t1), SG.pack_mask_frames(masks, DEV, t0, t1),
                       None, precision=N.PREC_TC, device=DEV)
    tr.params.copy_(params)
    tr.indices.copy_(inds)
    return tr


@pytest.mark.parametrize("it", [0, 6000], ids=["with_global", "without_global"])
def test_fullsize_trip_layers(fullsize, it, wg_units):
    """Whole video: the compacted flow groups have fewer live tiles than the ordinary groups, which are all live."""
    data, _, inds, _ = fullsize
    T, H, W, B = FULL["T"], FULL["H"], FULL["W"], FULL["B"]
    want = host_counts(inds, data, 0, T, H, W)
    n, nf, nb = want
    assert n == B and tiles_of(nf) < tiles_of(n) and tiles_of(nb) < tiles_of(n) and (nf % TM or nb % TM), want
    tr = _fullsize_trainer(fullsize, 0, T)
    run_trip(tr, it)
    check_trip(tr, it, want, wg_units, f"fullsize, {'with' if it == 0 else 'without'} the global term")


@pytest.mark.parametrize("world,rank", [(2, 0), (2, 1), (8, 0), (8, 7)])
def test_fullsize_shard_layers(fullsize, world, rank, wg_units):
    """One frame shard: counters[0] far below cap (most tiles of every group dead), compacted groups fewer still;
    rank 0's and the last rank's tile counts differ."""
    data, _, inds, _ = fullsize
    T, H, W, B = FULL["T"], FULL["H"], FULL["W"], FULL["B"]
    per_rank = []
    for r in (0, world - 1):
        n, nf, nb = host_counts(inds, data, *A.frame_range(r, world, T), H, W)
        per_rank.append((tiles_of(n), tiles_of(nf), tiles_of(nb)))
        assert tiles_of(nf) < tiles_of(n) < tiles_of(B) and tiles_of(nb) < tiles_of(n), (r, n, nf, nb)
    assert per_rank[0] != per_rank[1], per_rank
    t0, t1 = A.frame_range(rank, world, T)
    tr = _fullsize_trainer(fullsize, t0, t1)
    run_trip(tr, 0)
    check_trip(tr, 0, host_counts(inds, data, t0, t1, H, W), wg_units, f"{world}-way shard, rank {rank}")


# ---------------------------------------------------------------------------------------------------------------
# hand-built batches on a small video
# ---------------------------------------------------------------------------------------------------------------
def _small_trainer(data, masks, t0, t1, config=None, seed=7):
    cfg = {"samples_batch": B_SMALL}
    cfg.update(config or {})
    tr = SG.SegTrainer(A.DeviceVideo.from_reference_layout(data, DEV, t0, t1), SG.pack_mask_frames(masks, DEV, t0, t1),
                       cfg, precision=N.PREC_TC, device=DEV)
    torch.manual_seed(seed)
    tr.init_like_reference()
    return tr


@pytest.mark.parametrize("regime", ["no_fwd", "all_fwd", "fwd_whole_tiles"])
@pytest.mark.parametrize("n_local", [1, 127, 128, 129])
def test_small_batch_layers(n_local, regime, wg_units):
    _need_tc()
    n_f, n_b = flow_counts(n_local, regime)
    data, masks = small_data()
    T, H, W = SMALL["T"], SMALL["H"], SMALL["W"]
    t0, t1 = A.frame_range(0, 2, T)
    assert t0 <= FRAME < t1
    inds = small_batch(n_local, n_f, n_b, seed=n_local)
    want = host_counts(inds, data, t0, t1, H, W)
    assert want == (n_local, n_f, n_b), want
    # the TileIter edge of the regime
    if regime == "no_fwd":
        assert n_f == 0 and n_b > 0                                 # a compacted group with no tile at all
    elif regime == "all_fwd":
        assert n_f == n_local                                       # compacted group = ordinary group
    else:
        assert n_f % TM == 0 and n_b % TM != 0                      # a full last tile beside a partial one
    tr = _small_trainer(data, masks, t0, t1)
    tr.indices.copy_(inds)
    run_trip(tr, 0)
    check_trip(tr, 0, want, wg_units, f"small batch, n_local {n_local}, {regime} ({n_f} / {n_b} flow rows)")


def test_empty_shard_layers(wg_units):
    """Rank 1 of a 2-way split holds no sample of the batch: zero tiles run (every output row and image keeps the
    fill), the gradients are exactly zero, the weight images are still prepared."""
    _need_tc()
    data, masks = small_data()
    T, H, W = SMALL["T"], SMALL["H"], SMALL["W"]
    inds = FRAME * H * W + torch.randint(H * W, (B_SMALL,), generator=torch.Generator().manual_seed(9))
    t0, t1 = A.frame_range(1, 2, T)
    assert not t0 <= FRAME < t1
    tr = _small_trainer(data, masks, t0, t1)
    tr.indices.copy_(inds)
    run_trip(tr, 0)
    cnt = check_trip(tr, 0, (0, 0, 0), wg_units, "empty shard")
    assert cnt[1] > 0 and cnt[2] > 0                                 # the whole batch's flow counts are still there
    assert torch.count_nonzero(tr.grads) == 0


def test_cached_work_lists_layers(wg_units):
    """Two trips on one trainer (rank 0 of 2): the first eager (it caches the job tables and work lists, keyed on
    the row geometry), the second a CUDA-graph replay of a trip captured after it, on a batch with more resident
    rows but fewer forward-flow rows.  The second trip is checked layer by layer on the cached work lists."""
    _need_tc()
    data, masks = small_data()
    T, H, W = SMALL["T"], SMALL["H"], SMALL["W"]
    t0, t1 = A.frame_range(0, 2, T)
    first, second = (140, 130, 20), (300, 100, 250)
    assert tiles_of(second[0]) > tiles_of(first[0]) and tiles_of(second[1]) < tiles_of(first[1])
    tr = _small_trainer(data, masks, t0, t1)
    tr.indices.copy_(small_batch(*first, seed=1))
    run_trip(tr, 0)
    check_trip(tr, 0, first, wg_units, "cached work lists, first (eager) trip")
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        tr.loss_grad(0)
    tr.indices.copy_(small_batch(*second, seed=2))
    run_trip(tr, 0, replay=graph)
    check_trip(tr, 0, second, wg_units, "cached work lists, second (replayed) trip")


def test_pe_mappings_layers(wg_units):
    """use_positional_encoding_mapping1/2: both mappings on the position-encoded tensor-core kernels (4 and 2
    frequencies, 6 and 4 layers), whole video."""
    _need_tc()
    data, masks = small_data()
    T, H, W = SMALL["T"], SMALL["H"], SMALL["W"]
    tr = _small_trainer(data, masks, 0, T, {"use_positional_encoding_mapping1": True,
                                            "use_positional_encoding_mapping2": True})
    for which in ("mapping1", "mapping2"):
        assert N.lib().b200_mlp_tc_architecture(C.byref(tr.descs[which])) == 4, which
    inds = torch.randint(H * W * T, (B_SMALL,), generator=torch.Generator().manual_seed(4))
    tr.indices.copy_(inds)
    run_trip(tr, 0)
    want = host_counts(inds, data, 0, T, H, W)
    assert want[0] == B_SMALL and 0 < want[1] < B_SMALL
    check_trip(tr, 0, want, wg_units, "position-encoded mappings")


# ---------------------------------------------------------------------------------------------------------------
# the reconstruction
# ---------------------------------------------------------------------------------------------------------------
def _render_buffers(ws, rp):
    """plan_seg_render's carve of the render workspace (seg.cu): x_map, x3, uv1, uv2, ar, xat, yat as float views."""
    base = -ws.data_ptr() % 1024
    out, at = [], base
    for n, w in ((rp, 4), (rp, 3), (rp, 2), (rp, 2), (rp, 1), (2 * rp, 2), (2 * rp, 3)):
        out.append(ws[at:at + 4 * n * w].view(torch.float32).view(n, w))
        at += -(-4 * n * w // 256) * 256
    return out


def _seg_alpha(raw):
    f = np.float32
    return ((f(0.5) * (raw + f(1.0))) * f(0.99)) + f(0.001)


def test_seg_render_matches_training_forwards(fullsize):
    """b200_seg_render of frame 40 at 432 x 768 in chunks of 50 000 pixels (the last one not a multiple of 128): each
    network's inference output (no images stored) is bit-identical to a training-mode forward at the render's row
    counts (rp for the mappings and alpha, 2 rp for the atlas); the atlas input is seg_atlas_in's arithmetic; the
    composite, alpha and the 8-bit truncation equal their float32 restatement from those outputs bit for bit."""
    lib = N.lib()
    T, H, W = FULL["T"], FULL["H"], FULL["W"]
    _, _, _, params = fullsize
    tr = SG.SegTrainer(None, None, None, precision=N.PREC_TC, device=DEV, resx=W)
    tr.params.copy_(params)
    cfg = tr._config(0)
    f, chunk, HW = 40, 50000, H * W
    assert HW % chunk % TM != 0
    rgb = torch.empty(HW, 3, device=DEV)
    alpha = torch.empty(HW, device=DEV)
    u8 = torch.empty(HW, 3, dtype=torch.uint8, device=DEV)
    ws = torch.empty(int(lib.b200_seg_render_workspace_bytes(C.byref(cfg), chunk)), dtype=torch.uint8, device=DEV)
    st = N.current_stream()
    fp = lambda t: np.asarray(t.cpu().numpy(), dtype=np.float32)
    for p0 in range(0, HW, chunk):
        p1 = min(HW, p0 + chunk)
        count = p1 - p0
        rp = -(-count // TM) * TM
        N.check(lib.b200_seg_render(C.byref(cfg), N.ptr(tr.params), H, W, T, f, p0, p1, N.ptr(rgb[p0:]), N.ptr(u8[p0:]),
                                    N.ptr(alpha[p0:]), N.ptr(ws), ws.numel(), st), "b200_seg_render")
        torch.cuda.synchronize()
        _, x3, uv1, uv2, ar, xat, yat = _render_buffers(ws, rp)
        outs = {}
        for which, x, got in (("mapping1", x3, uv1), ("mapping2", x3, uv2), ("alpha", x3, ar), ("atlas", xat, yat)):
            d = tr.descs[which]
            rows = x.shape[0]
            y = torch.empty(rows, d.output_dim, device=DEV)
            nb = int(lib.b200_mlp_workspace_bytes(C.byref(d), rows, 1))
            tws = torch.empty(nb, dtype=torch.uint8, device=DEV)
            N.check(lib.b200_mlp_forward(C.byref(d), N.ptr(tr.params[tr.net_slice(which)]), N.ptr(x.clone()), N.ptr(y),
                                         rows, 1, N.PREC_TC, N.ptr(tws), nb, st), f"{which} training forward")
            torch.cuda.synchronize()
            assert torch.equal(y.view(torch.int32), got.view(torch.int32)), f"{which}: inference != training forward"
            outs[which] = fp(y)
        u1, u2 = outs["mapping1"], outs["mapping2"]
        want_xat = np.concatenate((u1 * np.float32(0.5) + np.float32(0.5), u2 * np.float32(0.5) - np.float32(0.5)))
        assert np.array_equal(fp(xat).view(np.int32), want_xat.view(np.int32)), "seg_atlas_in"
        a = _seg_alpha(outs["alpha"][:count, 0])
        y1, y2 = outs["atlas"][:count], outs["atlas"][rp:rp + count]
        c1 = (y1 + np.float32(1.0)) * np.float32(0.5)
        c2 = (y2 + np.float32(1.0)) * np.float32(0.5)
        o = c1 * a[:, None] + c2 * (np.float32(1.0) - a[:, None])
        assert np.array_equal(fp(alpha[p0:p1]).view(np.int32), a.view(np.int32)), f"alpha of pixels {p0}:{p1}"
        assert np.array_equal(fp(rgb[p0:p1]).view(np.int32), o.view(np.int32)), f"rgb of pixels {p0}:{p1}"
        want_u8 = np.trunc(o.astype(np.float64) * 255.0).astype(np.int64).astype(np.uint8)
        assert np.array_equal(u8[p0:p1].cpu().numpy(), want_u8), f"8-bit rgb of pixels {p0}:{p1}"
    print(f"seg render of frame {f}: {-(-HW // chunk)} chunks, every network output and the composite bit-exact")
