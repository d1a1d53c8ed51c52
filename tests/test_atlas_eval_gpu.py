"""Stage 1's reconstruction (b200_render_for) and evaluation maps (b200_eval_maps) at the benchmark geometry, 80 x 432 x
768 (synth.throughput_set, seed 0), with the oracle's final parameters of the full schedule at exactly this geometry
(tests/golden/quality_oracle.npz): uv spans the atlas and the rigidity values are those of a trained mapping.  The
position-encoded mapping (use_positional_encoding_mapping1 with 10 frequencies, network code 4) starts from
init_like_reference under a fixed seed, next to the same trained atlas.

Every call runs on a workspace whose buffers hold 0xFF (NaN) beforehand, and the buffers are read back through host
mirrors of the carves (b200_render_for in c_api.cu, plan_eval in eval_maps.cu), so padding rows must be written by the
kernels.  Frames are rendered / evaluated in chunks of 50 000 pixels (every chunk ends off a 128-row tile, and the
later ones start deep in the frame) and in one whole-frame call.

Render (tensor cores and fp32): the coordinate rows equal their fp32 restatement (norm_coord for x and y, the time
f / (T / 2.0) - 1 rounded once from double, evaluate.py:656); the inference forwards equal training-mode
b200_mlp_forward calls on the same rows bit for bit (the atlas on uv * 0.5 + 0.5 formed on the host: * 0.5 is exact,
so it is the operand of the kernel's in-kernel affine); rgb = (y + 1) * 0.5 in fp32 and u8 = trunc(float64(rgb) *
255) bit for bit; the chunked image equals the whole-frame image bit for bit.

Evaluation maps (both precisions, both mappings, frames 0, 1, 40, 78 and 79 = T - 1, forward masks as synthesised,
all zero and all one): the four row groups (x, y, t_render), (x, y - d, t), (x - d, y, t), (x + fx, y + fy, t + 1) and
the `valid` words equal their fp32 restatement bit for bit; the 4 x rp mapping outputs equal a training-mode forward
at 4 x rp rows bit for bit, and group 0 equals the render's uv of the same chunk bit for bit; the uv output is group 0;
rigidity and the forward flow error are restated in float64 from the device's own group outputs with the running-error
envelope of test_stage1_heads_gpu.py (C_ENV = 4); flow error is exactly 0 where the flow is invalid and on frame T - 1.
A frame-sharded video (frames [40, 80) resident) gives bit-identical maps for frames 40, 78 and 79.

CPU: the host mirror of plan_eval sizes the workspace as b200_eval_maps_workspace_bytes does; b200_seg_render and
b200_render_for refuse a frame outside the video.
"""
import ctypes as C
import os
import time

import numpy as np
import pytest
import torch

from b200 import _native as N
from b200 import atlas as A
from b200 import seg as SG
from b200 import synth
from csrc_build import ensure_built
from oracle import atlas_oracle as O
from tc_images_common import _need_tc
from test_stage1_heads_gpu import E, Ratios, _norm, _with_masks, flow, rigidity, vec

DEV = "cuda"
T, H, W = 80, 432, 768
HW = H * W
LARGER = max(H, W)
TM = 128
CHUNK = 50000
PE_FREQS = 10
ERR_INVALID, ERR_WORKSPACE = 1, 3                   # B200_ERR_INVALID, B200_ERR_WORKSPACE
HL, HT = np.float32(LARGER / 2.0), np.float32(T / 2.0)
RENDER_FRAMES = (0, 40, 79)
EVAL_FRAMES = (0, 1, 40, 78, 79)
EVAL_CHUNKED = (1, 78)                              # frames also evaluated in 50 000-pixel chunks
SHARD = (40, 80)
MAPPINGS = ("default", "pe")
PRECS = {"tc": N.PREC_TC, "fp32": N.PREC_FP32}
FIXTURE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "quality_oracle.npz")


def r256(n):
    return -(-n // 256) * 256


def rows_of(n):
    return -(-n // TM) * TM


def t_render(f):
    """evaluate.py:656: (f / (T / 2.0) - 1) in double, times an fp32 tensor of ones."""
    return np.float32(f / (T / 2.0) - 1.0)


def spans(chunked):
    return [(p0, min(HW, p0 + CHUNK)) for p0 in range(0, HW, CHUNK)] if chunked else [(0, HW)]


def bits(t):
    return t.contiguous().view(torch.int32)


def host(t):
    return t.detach().cpu().numpy()


# ---------------------------------------------------------------------------------------------------------------
# host mirrors of the workspace carves
# ---------------------------------------------------------------------------------------------------------------
def scratch_layout(desc, rows):
    """plan_mlp_scratch (c_api.cu): (offset of the output buffer y, total bytes) of one network's fp32 scratch."""
    dims = A.layer_dims(desc)
    off = 0
    for l, (k, _) in enumerate(dims):
        if l == 0 and desc.pe_freqs == 0:
            continue
        off += r256(rows * k * 4)
    y_off = off
    off += r256(rows * desc.output_dim * 4)
    wz = max(desc.hidden_dim, dims[0][0], desc.output_dim)
    return y_off, off + 2 * r256(rows * wz * 4)


def render_views(ws, rows, prec, mdesc, adesc):
    """b200_render_for's carve from the 256-aligned base: x_map [rows][4]; then uv [rows][2] and y [rows][3] on the
    tensor cores, or the mapping's and the atlas's plan_mlp_scratch in fp32 (uv and y are their output buffers)."""
    at = -ws.data_ptr() % 256

    def view(off, w):
        assert off + 4 * rows * w <= ws.numel()
        return ws[off:off + 4 * rows * w].view(torch.float32).view(rows, w)
    x_map = view(at, 4)
    at += r256(rows * 16)
    if prec == N.PREC_TC:
        return x_map, view(at, 2), view(at + r256(rows * 8), 3)
    y_m, tot_m = scratch_layout(mdesc, rows)
    y_a, _ = scratch_layout(adesc, rows)
    return x_map, view(at + y_m, 2), view(at + tot_m + y_a, 3)


def eval_layout(lib, desc, pixels):
    """plan_eval (eval_maps.cu): rows_pad, the byte offsets of x3 [4][rp][3], valid [rp], uv [4][rp][2] and of the
    mapping call's workspace, and the plan's size, relative to its 1024-aligned base."""
    rp = rows_of(pixels)
    need = int(lib.b200_mlp_workspace_bytes(C.byref(desc), 4 * rp, 0))
    assert need > 0
    o_x3 = 0
    o_valid = o_x3 + r256(4 * rp * 12)
    o_uv = o_valid + r256(rp * 4)
    o_ws = o_uv + r256(4 * rp * 8)
    return rp, o_x3, o_valid, o_uv, o_ws, o_ws + r256(-(-need // 1024) * 1024 + 1024)


def eval_views(lib, desc, ws, pixels):
    rp, o_x3, o_valid, o_uv, _, _ = eval_layout(lib, desc, pixels)
    base = -ws.data_ptr() % 1024
    f = lambda o, n: ws[base + o:base + o + 4 * n].view(torch.float32)
    return rp, f(o_x3, 4 * rp * 3).view(4, rp, 3), f(o_valid, rp), f(o_uv, 4 * rp * 2).view(4, rp, 2)


# ---------------------------------------------------------------------------------------------------------------
# fp32 restatements
# ---------------------------------------------------------------------------------------------------------------
def render_rows(f, p0, p1, rows):
    p = np.arange(p0, p1)
    out = np.zeros((rows, 4), np.float32)
    out[:p.size, 0] = _norm((p % W).astype(np.float32), HL)
    out[:p.size, 1] = _norm((p // W).astype(np.float32), HL)
    out[:p.size, 2] = t_render(f)
    return out


def eval_rows(data, f, p0, p1, rp, d):
    """eval_rows_kernel in fp32: the four row groups and the valid words of pixels [p0, p1) of frame f."""
    p = np.arange(p0, p1)
    n = p.size
    fx, fy = (p % W).astype(np.float32), (p // W).astype(np.float32)
    fl = data["flow_fwd"][:, :, :, f, 0].numpy().reshape(HW, 2)[p]
    ok = data["mask_fwd"][:, :, f, 0].numpy().reshape(HW)[p] != 0
    ft = np.full(n, f, np.float32)
    tn = _norm(ft, HT)
    rows = np.zeros((4, rp, 3), np.float32)
    rows[0, :n] = np.stack([_norm(fx, HL), _norm(fy, HL), np.full(n, t_render(f))], axis=1)
    rows[1, :n] = np.stack([_norm(fx, HL), _norm(fy - d, HL), tn], axis=1)
    rows[2, :n] = np.stack([_norm(fx - d, HL), _norm(fy, HL), tn], axis=1)
    rows[3, :n] = np.stack([_norm(fx + fl[:, 0], HL), _norm(fy + fl[:, 1], HL), _norm(ft + np.float32(1.0), HT)], axis=1)
    valid = np.zeros(rp, np.float32)
    valid[:n] = ok
    return rows, valid


# ---------------------------------------------------------------------------------------------------------------
# fixtures and calls
# ---------------------------------------------------------------------------------------------------------------
class Scratch:
    """Device buffers reused between calls (the whole-frame fp32 workspaces are several GB)."""

    def __init__(self):
        self.b = {}

    def __call__(self, name, nbytes):
        t = self.b.get(name)
        if t is None or t.numel() < nbytes:
            self.b.pop(name, None)
            t = self.b[name] = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
        return t[:nbytes]


def _unflat(spec, flat):
    out, off = [], 0
    for k, n in spec.layer_dims():
        out += [torch.from_numpy(flat[off:off + k * n]).view(n, k)]
        off += k * n
        out += [torch.from_numpy(flat[off:off + n])]
        off += n
    return O.state_dict_of(out)


@pytest.fixture(scope="module")
def data():
    return synth.throughput_set(H, W, T, seed=0)


@pytest.fixture(scope="module")
def trainers():
    """Parameters of both mappings in AtlasTrainers without a video (only their flat parameters are used)."""
    fx = np.load(FIXTURE)
    assert tuple(int(v) for v in fx["video"]) == (T, H, W)
    map_sd, atl_sd = _unflat(O.MAPPING_SPEC, fx["mapping_params"]), _unflat(O.ATLAS_SPEC, fx["atlas_params"])
    out = {}
    tr = A.AtlasTrainer(None, precision=N.PREC_TC, device=DEV)
    tr.load_state(map_sd, atl_sd)
    out["default"] = tr
    tr = A.AtlasTrainer(None, {"use_positional_encoding_mapping1": True,
                               "number_of_positional_encoding_mapping1": PE_FREQS}, precision=N.PREC_TC, device=DEV)
    torch.manual_seed(11)
    tr.init_like_reference()
    tr.load_state(tr.state_dict("mapping"), atl_sd)
    assert N.lib().b200_mlp_tc_architecture(C.byref(tr.map_desc)) == 4
    out["pe"] = tr
    return out


@pytest.fixture(scope="module")
def videos(data):
    """Whole-video DeviceVideos per mask mode, and the mixed-mask video resident on frames [40, 80) only; built on
    first use."""
    cache = {}

    def get(mode, shard=False):
        key = (mode, shard)
        if key not in cache:
            cache[key] = A.DeviceVideo.from_reference_layout(_with_masks(data, mode), DEV, *(SHARD if shard else (0, T)))
        return cache[key]
    yield get
    cache.clear()
    torch.cuda.empty_cache()


@pytest.fixture(scope="module")
def scratch():
    s = Scratch()
    yield s
    s.b.clear()
    torch.cuda.empty_cache()


def training_forward(lib, scratch, desc, params, x, prec):
    """Stand-alone b200_mlp_forward in training mode on the rows of x."""
    rows = x.shape[0]
    x = x.contiguous()
    y = torch.empty(rows, desc.output_dim, device=DEV)
    nb = int(lib.b200_mlp_workspace_bytes(C.byref(desc), rows, 1))
    ws = scratch("forward", nb)
    N.check(lib.b200_mlp_forward(C.byref(desc), N.ptr(params), N.ptr(x), N.ptr(y), rows, 1, prec, N.ptr(ws), nb,
                                 N.current_stream()), "training forward")
    torch.cuda.synchronize()
    return y


def render_chunk(lib, scratch, tr, prec, f, p0, p1, rgb, u8):
    """One b200_render_for call on a 0xFF workspace; returns the views (x_map, uv, y) of its buffers."""
    md = C.byref(tr.map_desc)
    nb = int(lib.b200_render_workspace_bytes_for(md, p1 - p0))
    ws = scratch("render", nb)
    ws.fill_(0xFF)
    N.check(lib.b200_render_for(md, N.ptr(tr.params), H, W, T, f, p0, p1, N.ptr(rgb[p0:]), N.ptr(u8[p0:]), prec,
                                N.ptr(ws), nb, N.current_stream()), "b200_render_for")
    torch.cuda.synchronize()
    return render_views(ws, rows_of(p1 - p0), prec, tr.map_desc, tr.atlas_desc)


# ---------------------------------------------------------------------------------------------------------------
# 1, 2: the render
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("mapping", MAPPINGS)
@pytest.mark.parametrize("prec", list(PRECS), ids=list(PRECS))
def test_render_matches_training_forwards(trainers, scratch, prec, mapping):
    """b200_render_for of frames 0, 40 and 79, in 50 000-pixel chunks and in one call.  Bound: bit-exact, every
    buffer.  x_map: fp32 restatement, padding rows zero.  uv: training-mode b200_mlp_forward(mapping) on the x_map
    rows at the render's row count.  y: training-mode b200_mlp_forward(atlas) on uv * 0.5 + 0.5 formed on the host.
    On the tensor cores the inference kernels run without their image stores, on a job table rebuilt per call, with
    the atlas affine inside the kernel; in fp32, the affine sits in the encoding kernel.  rgb = (y + 1) * 0.5 in fp32,
    u8 = trunc(float64(rgb) * 255).  The chunked image equals the whole-frame image."""
    if PRECS[prec] == N.PREC_TC:
        _need_tc()
    p_ = PRECS[prec]
    lib = N.lib()
    tr = trainers[mapping]
    assert HW % CHUNK % TM and CHUNK % TM
    pm, pa = tr.params[tr.net_slice("mapping")], tr.params[tr.net_slice("atlas")]
    half, one = np.float32(0.5), np.float32(1.0)
    t0 = time.time()
    n_calls = 0
    for f in RENDER_FRAMES:
        images = []
        for chunked in (True, False):
            rgb = torch.full((HW, 3), float("nan"), device=DEV)
            u8 = torch.zeros((HW, 3), dtype=torch.uint8, device=DEV)
            for p0, p1 in spans(chunked):
                n, rows = p1 - p0, rows_of(p1 - p0)
                x_map, uv, y = render_chunk(lib, scratch, tr, p_, f, p0, p1, rgb, u8)
                n_calls += 1
                where = f"{prec} {mapping} frame {f} pixels [{p0}, {p1})"
                want_x = render_rows(f, p0, p1, rows)
                assert np.array_equal(host(x_map).view(np.int32), want_x.view(np.int32)), f"{where}: x_map"
                want_uv = training_forward(lib, scratch, tr.map_desc, pm, x_map[:, :3], p_)
                assert torch.equal(bits(uv), bits(want_uv)), f"{where}: uv != training forward"
                uv_h = host(uv)
                x_at = torch.from_numpy(uv_h * half + half).to(DEV)
                want_y = training_forward(lib, scratch, tr.atlas_desc, pa, x_at, p_)
                assert torch.equal(bits(y), bits(want_y)), f"{where}: y != training forward"
                o = (host(y)[:n] + one) * half
                assert np.array_equal(host(rgb[p0:p1]).view(np.int32), o.view(np.int32)), f"{where}: rgb"
                want_u8 = np.trunc(o.astype(np.float64) * 255.0).astype(np.uint8)
                assert np.array_equal(host(u8[p0:p1]), want_u8), f"{where}: u8"
            images.append((rgb, u8))
        (rc, uc), (rw, uw) = images
        assert torch.equal(bits(rc), bits(rw)) and torch.equal(uc, uw), f"{prec} {mapping} frame {f}: chunked != whole"
    print(f"\n[render {prec} {mapping}] frames {RENDER_FRAMES}, {n_calls} calls: x_map, uv, y, rgb, u8 and chunked "
          f"vs whole frame bit-exact ({time.time() - t0:.1f} s)")


# ---------------------------------------------------------------------------------------------------------------
# 3: the evaluation maps
# ---------------------------------------------------------------------------------------------------------------
def eval_call(lib, scratch, tr, vid, prec, f, p0, p1, uv, rig, fl):
    """One b200_eval_maps call whose x3 / valid / uv buffers hold 0xFF beforehand; returns (rp, x3, valid, uv4)."""
    md = C.byref(tr.map_desc)
    nb = int(lib.b200_eval_maps_workspace_bytes(md, p1 - p0))
    ws = scratch("eval", nb)
    ws[:-ws.data_ptr() % 1024 + eval_layout(lib, tr.map_desc, p1 - p0)[4]].fill_(0xFF)      # x3, valid, uv
    N.check(lib.b200_eval_maps(md, N.ptr(tr.params[tr.net_slice("mapping")]), C.byref(vid.struct), f, p0, p1,
                               float(tr.cfg["derivative_amount"]), float(tr.cfg["uv_mapping_scale"]), prec, N.ptr(uv[p0:]),
                               N.ptr(rig[p0:]), N.ptr(fl[p0:]), N.ptr(ws), nb, N.current_stream()), "b200_eval_maps")
    torch.cuda.synchronize()
    return eval_views(lib, tr.map_desc, ws, p1 - p0)


def check_heads(rt, u4, valid, rig, fl, f, n):
    """rigidity and flow error of a whole frame in float64 from the device's group outputs u4 [4][>= n][2]; returns
    the undecidable sample counts."""
    L, s, d = float(LARGER), float(np.float32(0.8)), 1.0
    U = [vec(u4[g, :n]) for g in range(4)]
    zero = lambda: [E(np.zeros(n)), E(np.zeros(n))]
    und_r = np.zeros(n, bool)
    ref_r = rigidity(U[0], U[1], U[2], L, s, d, 0.0, zero(), zero(), zero(), und_r)
    rt.close("rigidity", rig, ref_r, ~und_r)
    on = valid[:n] != 0
    if f == T - 1:
        assert np.all(fl == 0.0), "flow error of the last frame is not 0"
        return int(und_r.sum()), 0
    und_f = np.zeros(n, bool)
    ref_f = flow(U[0], U[3], L, s, 0.0, zero(), zero(), und_f, on)
    rt.close("flow_error", fl, ref_f, on & ~und_f)
    assert np.all(fl[~on] == 0.0), "flow error where the flow is invalid is not 0"
    return int(und_r.sum()), int(und_f.sum())


@pytest.mark.gpu
@pytest.mark.parametrize("mapping", MAPPINGS)
@pytest.mark.parametrize("prec", list(PRECS), ids=list(PRECS))
def test_eval_maps_rows_outputs_and_heads(data, trainers, videos, scratch, prec, mapping):
    """b200_eval_maps of frames 0, 1, 40, 78, 79 under three forward-mask modes (synthesised, all zero, all one); frames
    1 and 78 also in 50 000-pixel chunks.  Bit-exact: the x3 rows and valid words against their fp32 restatement
    (padding rows zero); the 4 x rp mapping outputs against a training-mode b200_mlp_forward at 4 x rp rows; group 0
    against b200_render_for's uv of the same chunk; the uv output against group 0; chunked maps against whole-frame
    maps; the maps of frames 40, 78, 79 of a video resident on frames [40, 80) against the whole video's.  Envelope:
    rigidity and flow error (on the valid rows) within C_ENV * u * envelope of float64 from the device's own group
    outputs (test_stage1_heads_gpu.py, C_ENV = 4); undecidable samples only finite.  Flow error exactly 0 on invalid
    rows and on frame T - 1."""
    if PRECS[prec] == N.PREC_TC:
        _need_tc()
    p_ = PRECS[prec]
    lib = N.lib()
    tr = trainers[mapping]
    d = np.float32(tr.cfg["derivative_amount"])
    pm = tr.params[tr.net_slice("mapping")]
    rt = Ratios(f"eval maps {prec} {mapping}")
    rgb = torch.empty((HW, 3), device=DEV)                              # the render's outputs (unchecked here)
    u8 = torch.empty((HW, 3), dtype=torch.uint8, device=DEV)
    t0 = time.time()
    whole = {}
    und = []
    for mode in ("mixed", "zero", "one"):
        md = _with_masks(data, mode)
        vid = videos(mode)
        for f in EVAL_FRAMES:
            maps = []
            for chunked in ((True, False) if f in EVAL_CHUNKED else (False,)):
                uv = torch.full((HW, 2), float("nan"), device=DEV)
                rig = torch.full((HW,), float("nan"), device=DEV)
                fl = torch.full((HW,), float("nan"), device=DEV)
                for p0, p1 in spans(chunked):
                    n = p1 - p0
                    where = f"{prec} {mapping} masks {mode} frame {f} pixels [{p0}, {p1})"
                    rp, x3, valid, u4 = eval_call(lib, scratch, tr, vid, p_, f, p0, p1, uv, rig, fl)
                    want_rows, want_valid = eval_rows(md, f, p0, p1, rp, d)
                    assert np.array_equal(host(x3).view(np.int32), want_rows.view(np.int32)), f"{where}: x3 rows"
                    assert np.array_equal(host(valid).view(np.int32), want_valid.view(np.int32)), f"{where}: valid"
                    want_u4 = training_forward(lib, scratch, tr.map_desc, pm, x3.reshape(4 * rp, 3), p_)
                    assert torch.equal(bits(u4.reshape(4 * rp, 2)), bits(want_u4)), f"{where}: mapping outputs"
                    _, r_uv, _ = render_chunk(lib, scratch, tr, p_, f, p0, p1, rgb, u8)
                    assert torch.equal(bits(u4[0]), bits(r_uv)), f"{where}: group 0 != the render's uv"
                    assert torch.equal(bits(uv[p0:p1]), bits(u4[0, :n])), f"{where}: uv output != group 0"
                    if not chunked:
                        u4_h, valid_h = host(u4), host(valid)
                maps.append((uv, rig, fl))
            if len(maps) == 2:
                for a, b in zip(*maps):
                    assert torch.equal(bits(a), bits(b)), f"{prec} {mapping} masks {mode} frame {f}: chunked != whole"
            uv, rig, fl = maps[-1]
            und.append(check_heads(rt, u4_h, valid_h, host(rig), host(fl), f, HW))
            if mode == "mixed":
                whole[f] = maps[-1]
    # the frame-sharded video: record offset frame - t_begin
    vid = videos("mixed", shard=True)
    for f in (40, 78, 79):
        got = [torch.full_like(t, float("nan")) for t in whole[f]]
        eval_call(lib, scratch, tr, vid, p_, f, 0, HW, *got)
        for a, b in zip(got, whole[f]):
            assert torch.equal(bits(a), bits(b)), f"{prec} {mapping} frame {f}: frame shard [40, 80) != whole video"
    print(f"\n[eval maps {prec} {mapping}] rows, valid, mapping outputs, group 0 = render uv, uv output, chunking and "
          f"the frame shard bit-exact; undecidable samples per case (rigidity, flow): {und} "
          f"({time.time() - t0:.1f} s)")
    assert rt.report() <= 1.0


# ---------------------------------------------------------------------------------------------------------------
# CPU: the workspace mirror, the frame checks
# ---------------------------------------------------------------------------------------------------------------
def test_eval_workspace_mirror_matches_the_library():
    """The host mirror of plan_eval, plus the 2048 bytes of alignment slack, is b200_eval_maps_workspace_bytes exactly,
    for both mappings at tile edges, the chunk sizes of the GPU tests and a whole frame."""
    ensure_built()
    lib = N.lib()
    for pe in (0, PE_FREQS):
        desc = A.make_desc(**dict(A.MAPPING_DESC, pe_freqs=pe))
        for pixels in (1, 127, 128, 129, CHUNK, HW % CHUNK, HW):
            assert eval_layout(lib, desc, pixels)[5] + 2048 == lib.b200_eval_maps_workspace_bytes(C.byref(desc), pixels), \
                (pe, pixels)


def test_renders_refuse_a_frame_outside_the_video():
    """b200_seg_render, like b200_render_for, refuses frame >= T (and frame < 0) with B200_ERR_INVALID and a message,
    before any device work; frame T - 1 passes that check and is refused only for its empty workspace."""
    ensure_built()
    lib = N.lib()
    d = SG.seg_descs(SG.SEG_DEFAULTS)
    cfg = N.SegConfig(10000, 1, N.PREC_FP32, W, 0.8, 1.0, 100.0, 5000.0, 1000.0, 1.0, 5.0, 50.0, 500.0, 4900.0, 1000.0,
                      2000.0, d["mapping1"], d["mapping2"], d["alpha"], d["atlas"])
    buf = (C.c_float * 64)()
    p = C.cast(buf, C.c_void_p)
    md = A.make_desc(**A.MAPPING_DESC)
    for frame in (T, T + 1, -1):
        assert lib.b200_seg_render(C.byref(cfg), p, H, W, T, frame, 0, HW, p, None, p, p, 1 << 40, None) == ERR_INVALID
        assert f"frame {frame} is outside".encode() in lib.b200_last_error()
        assert lib.b200_render_for(C.byref(md), p, H, W, T, frame, 0, HW, p, None, N.PREC_FP32, p, 1 << 40,
                                   None) == ERR_INVALID
        assert b"bad render range" in lib.b200_last_error()
    assert lib.b200_seg_render(C.byref(cfg), p, H, W, T, T - 1, 0, HW, p, None, p, p, 0, None) == ERR_WORKSPACE
    assert lib.b200_render_for(C.byref(md), p, H, W, T, T - 1, 0, HW, p, None, N.PREC_FP32, p, 0, None) == ERR_WORKSPACE
