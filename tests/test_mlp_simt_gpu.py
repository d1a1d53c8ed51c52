"""The fp32 CUDA-core IMLP path (B200_PREC_FP32: `sgemm_kernel` and `out_grad_kernel` of csrc/mlp_simt.cu, the
positional-encoding kernels of csrc/atlas_kernels.cu, `plan_mlp_scratch` / `mlp_forward_impl` / `mlp_backward_impl` of
csrc/c_api.cu) one layer at a time against float64, at the shapes the configs and the `IMLP` class accept.  This path
runs every network that has no tensor-core kernels (any width but 256, other depths, PE counts or skips) and is the
cross-check of the tensor-core path.

Each case calls b200_mlp_forward / b200_mlp_backward through the C ABI with a workspace the test owns (filled with NaN
bytes, so that a read of an unwritten scratch element shows), then reads the device's own intermediates from it: the
input of every layer act[l] (post-ReLU, skip part appended), the output y and the last gradient buffer dz.  A mirror of
`plan_mlp_scratch` (`plan` below) locates them; a CPU test pins the mirror to b200_mlp_workspace_bytes.

The references are operand-exact: every layer is recomputed in float64 from the device's own fp32 operands, so no
ReLU mask can differ between the two sides.  With u = 2^-24, c = C_FP32 and |.| taken element-wise:

  forward, layer l (fan-in K):  z = act[l] W_l^T + b_l
      |act[l+1] - relu(z)|, |y - tanh(z)| or |y - z|  <=  c u sqrt(K) (|act[l]| |W_l|^T) + 4u (|b_l| + |z|)
                                                          (+ 4u |y| for tanhf, which is within 2 ulp)
  encoding:  act[0] against float64 sin / cos of the same fp32 products x b_k:  <= 4u |ref| (sinf / cosf are within
      2 ulp over the whole range); every skip slot is a bit-identical copy of act[0] (PE) or of x (no PE).
  backward:  G_{L-1} = dy (1 - y^2) with the device's y (or dy without tanh), error envelope E_{L-1} = 4u |dy| (1 + y^2)
      (or 0), then through every layer l > 0 of fan-out N_l, with the device's mask M_l = (act[l][:, :hidden] > 0):
          G_{l-1} = (G_l W_l[:, :hidden]) M_l
          E_{l-1} = M_l (E_l |W_l[:, :hidden]| + c u sqrt(N_l) |G_l| |W_l[:, :hidden]|)
      The device's last gradient buffer (G_0) is held to E_0.
  weight / bias gradients (split over rows in chunks of 1024, sequential FMA inside a chunk, one fp32 atomic per
      chunk):  |dW_l - G_l^T A_l| <= E_l^T |A_l| + c u (sqrt(min(rows, 1024)) + ceil(rows / 1024)) |G_l|^T |A_l|,
      db_l likewise with A_l = 1.  A_l is act[l], or x for layer 0 without encoding.
  input gradient:  dx = G_0 W_0 (no encoding) or, through the encoding, d_enc = G_0 W_0 followed by
      dx_j = sum_k b_k (ds_kj c_kj - dc_kj s_kj) on the device's s, c:
          |d_enc - ref| <= E_enc = E_0 |W_0| + c u sqrt(N_0) |G_0| |W_0|
          |dx - ref| <= sum_k b_k (E_enc,s |c| + E_enc,c |s|) + c u (2 + F) sum_k b_k (|ds c| + |dc s|)

c = 4, as in tests/test_conv_kernels_gpu.py.  Every case prints its worst ratio of error to bound (`pytest -s`).  On an
H100 80GB HBM3 at a 400 W power limit the largest was 0.48, for the encoding (about 1 ulp against the 2-ulp bound); the
largest GEMM ratio was 0.25 (a hidden activation), so the GEMM bounds hold with c = 1 and c = 4 leaves a 4x margin.
None of the ratios grows with the fan-in (0.18-0.25 from K = 1 to 512) or with the row count (up to 100 000 rows).

Every case of the table names the branch it exists for.  The last part of the file runs the segmentation trip with a
configuration in which some networks leave the tensor cores."""
import ctypes as C
import math
import zlib

import numpy as np
import pytest
import torch

from b200 import _native as N
from b200 import atlas as A
from b200 import seg as SG
from oracle import atlas_oracle as O
from oracle import seg_oracle as S
from seg_common import ORDER, load_fixture

DEV = "cuda"
U = 2.0 ** -24
C_FP32 = 4.0
ROW_CHUNK = 1024          # the weight gradient's split over rows (simt_mlp_backward)


def _r256(v):
    return (v + 255) // 256 * 256


def _ceil128(v):
    return (v + 127) // 128 * 128


# ---------------------------------------------------------------------------------------------------------------
# Mirror of resolve_mlp + plan_mlp_scratch (csrc/c_api.cu): byte offsets from the workspace base rounded up to 256
# ---------------------------------------------------------------------------------------------------------------
def plan(desc, rows):
    L, pe = desc.num_layers, desc.pe_freqs
    enc = 2 * desc.input_dim * pe if pe > 0 else desc.input_dim
    skip = [l > 0 and bool((desc.skip_mask >> l) & 1) for l in range(L)]
    K = [enc if l == 0 else desc.hidden_dim + (enc if skip[l] else 0) for l in range(L)]
    Nn = [desc.output_dim if l == L - 1 else desc.hidden_dim for l in range(L)]
    rp = _ceil128(rows)
    off, act = 0, []
    for l in range(L):
        if l == 0 and pe == 0:
            act.append(None)
            continue
        act.append(off)
        off += _r256(rp * K[l] * 4)
    y = off
    off += _r256(rp * desc.output_dim * 4)
    wz = max(desc.hidden_dim, enc, desc.output_dim)
    dz = [off, off + _r256(rp * wz * 4)]
    off = dz[1] + _r256(rp * wz * 4)
    return dict(act=act, y=y, dz=dz, total=off, K=K, N=Nn, enc=enc, skip=skip)


# ---------------------------------------------------------------------------------------------------------------
# Case table
# ---------------------------------------------------------------------------------------------------------------
CASES = {}


def _case(name, branch, in_dim=3, out_dim=2, hidden=48, layers=4, pe=0, skips=(), tanh=True, rows=300, x_offset=0,
          accumulate=False):
    CASES[name] = dict(name=name, branch=branch, in_dim=in_dim, out_dim=out_dim, hidden=hidden, layers=layers, pe=pe,
                       skips=tuple(skips), tanh=tanh, rows=rows, x_offset=x_offset, accumulate=accumulate)


# hidden width: 128-column J tiles of sgemm_kernel, float4 against scalar tile loads (ld % 4, pointer alignment)
_case("hidden1", "width 1: every tile ragged, scalar loads everywhere", hidden=1)
_case("hidden3", "width 3: scalar loads, output as wide as the hidden layer", in_dim=2, out_dim=3, hidden=3, layers=5)
_case("hidden100", "ld 100 (float4) and 103 on the skip layer (scalar) in one network", hidden=100, skips=(2,), rows=1025)
_case("hidden128", "exactly one J tile", hidden=128, layers=5, rows=1025)
_case("hidden129", "a one-column second J tile", hidden=129)
_case("hidden130", "ld 130 % 4 = 2: scalar loads of every hidden operand", hidden=130, skips=(2,))
_case("hidden256_depth5", "the stage-1 width on a depth without tensor-core kernels", hidden=256, layers=5, rows=1025)
_case("hidden384", "three J tiles", hidden=384, layers=3, rows=600)
_case("hidden512", "four J tiles", hidden=512, layers=3, rows=1025)
# input / output widths
for _d in (1, 2, 3, 5):
    _case(f"in{_d}", f"input width {_d}: scalar loads of x", in_dim=_d, hidden=32)
_case("in4", "input width 4: float4 loads of x", in_dim=4, hidden=32)
_case("in4_misaligned", "x at base + 1 float: the unaligned scalar fallback of load_tile", in_dim=4, hidden=32, x_offset=1)
for _d in (1, 2, 3, 7):
    _case(f"out{_d}", f"output width {_d}", out_dim=_d, hidden=32)
# 100 000 rows: 782 I tiles, so the last layer's input-gradient tiles that read the overlap run after the tiles that
# overwrote it (with a few tiles, all of them load before any stores and the overlap went unseen)
_case("out3_hidden2", "output wider than hidden and input, within 2x: the dz ping-pong buffers overlapped",
      in_dim=2, out_dim=3, hidden=2, layers=3, rows=100000)
_case("out7_hidden2", "output more than twice as wide: the output gradient overran the scratch",
      in_dim=1, out_dim=7, hidden=2, layers=3)
# positional encoding: pe_forward_kernel / pe_backward_kernel
_case("pe1_in1", "1 frequency, input width 1", in_dim=1, pe=1, hidden=32)
_case("pe5_in2", "5 frequencies, input width 2", in_dim=2, pe=5, hidden=32)
_case("pe10_in3", "10 frequencies, input width 3", in_dim=3, pe=10, hidden=32)
_case("pe16_in2", "16 frequencies: past the reference configs' 10", in_dim=2, pe=16, hidden=32)
_case("pe30_in1", "30 frequencies: the largest the library takes (arguments up to 2^29 pi)", in_dim=1, pe=30, hidden=32)
_case("pe_skip1", "PE with one skip layer", in_dim=2, pe=4, layers=6, skips=(3,))
_case("pe_skip2", "PE with skips 4 and 7 (the atlas pattern) at width 64", in_dim=2, pe=4, hidden=64, layers=8,
      skips=(4, 7))
_case("pe_skip3", "PE with three skip layers, one of them layer 1", in_dim=3, pe=3, layers=6, skips=(1, 3, 5))
# skips without encoding: the raw input copied by cudaMemcpy2DAsync
_case("skips_4_6", "skips 4 and 6 at 8 layers (the IMLP default)", hidden=64, layers=8, skips=(4, 6))
_case("skip_output", "a skip on the output layer", hidden=64, layers=8, skips=(4, 7))
_case("skip_layer1", "a skip on layer 1", skips=(1,))
_case("skips_consecutive", "consecutive skips", layers=6, skips=(2, 3))
_case("skips_five", "five skips (no limit without encoding)", layers=8, skips=(1, 2, 3, 5, 6))
_case("skip_beyond_depth", "skip indices >= num_layers are ignored, as in the reference", layers=6, skips=(2, 6, 9))
# depth
_case("depth2", "two layers: input layer straight into the output layer", layers=2)
_case("depth16", "sixteen layers (B200_MAX_LAYERS)", layers=16, hidden=40)
# output activation
_case("no_tanh", "use_tanh=False: out_grad_kernel copies dy", tanh=False)
_case("no_tanh_pe", "use_tanh=False with an encoding", in_dim=2, pe=3, tanh=False)
# rows: 128-row I tiles and the weight gradient's 1024-row chunks
for _r in (1, 3, 127, 128, 129, 1023, 1024, 1025, 2049):
    _case(f"rows{_r}", f"{_r} rows", rows=_r)
_case("rows70000", "69 weight-gradient chunks: many atomics per weight", hidden=8, layers=3, rows=70000)
_case("pe_rows2049", "three weight-gradient chunks with an encoding and a skip", in_dim=2, pe=2, layers=5, skips=(2,),
      rows=2049)
# accumulation: the header says dparams +=
_case("accumulate", "two backward calls into one gradient buffer", in_dim=2, pe=2, layers=5, skips=(2,), rows=2049,
      accumulate=True)


def _desc(c):
    return A.make_desc(c["in_dim"], c["out_dim"], c["hidden"], c["layers"], c["pe"], c["skips"], c["tanh"])


def _seed(name):
    return zlib.crc32(name.encode()) & 0x7FFFFFFF


def _inputs(c, total, desc):
    """He-uniform weights (activations keep their scale through 16 layers), nn.Linear-sized biases, x in [-1, 1]."""
    g = torch.Generator().manual_seed(_seed(c["name"]))
    w_off, b_off, _ = A.mlp_layout(desc)
    flat = torch.zeros(total)
    for i, (k, n) in enumerate(A.layer_dims(desc)):
        flat[w_off[i]:w_off[i] + k * n] = (torch.rand(n * k, generator=g) * 2 - 1) * math.sqrt(6.0 / k)
        flat[b_off[i]:b_off[i] + n] = (torch.rand(n, generator=g) * 2 - 1) / math.sqrt(k)
    x = torch.rand(c["rows"], c["in_dim"], generator=g) * 2 - 1
    dy = torch.randn(c["rows"], c["out_dim"], generator=g)
    return flat, x, dy


def _freqs(pe):
    return torch.tensor([(2 ** k) * np.pi for k in range(pe)], dtype=torch.float32)   # pe_freq(k), rounded to fp32


class Run:
    """One forward + backward call and the device's intermediates read back from the workspace."""

    def __init__(self, c):
        lib = N.lib()
        self.c, self.desc = c, _desc(c)
        self.w_off, self.b_off, self.total = A.mlp_layout(self.desc)
        rows = c["rows"]
        self.plan = pl = plan(self.desc, rows)
        flat, x, dy = _inputs(c, self.total, self.desc)
        extra = rows * pl["enc"] * 4 if c["pe"] else 0          # the encoded-input gradient of the PE backward
        nbytes = int(lib.b200_mlp_workspace_bytes(C.byref(self.desc), rows, 1)) + extra
        self.ws = torch.full((nbytes,), 0xFF, dtype=torch.uint8, device=DEV)    # NaN in every float
        self.base = _r256(self.ws.data_ptr()) - self.ws.data_ptr()
        xbuf = torch.full((rows * c["in_dim"] + c["x_offset"],), float("nan"), device=DEV)
        xbuf[c["x_offset"]:] = x.to(DEV).flatten()
        self.x = xbuf[c["x_offset"]:].view(rows, c["in_dim"])
        self.flat, self.dy = flat.to(DEV), dy.to(DEV)
        self.y = torch.full((rows, c["out_dim"]), float("nan"), device=DEV)
        self.dparams = torch.zeros(self.total, device=DEV)
        self.dx = torch.full((rows, c["in_dim"]), float("nan"), device=DEV)
        st = N.current_stream()
        N.check(lib.b200_mlp_forward(C.byref(self.desc), N.ptr(self.flat), N.ptr(self.x), N.ptr(self.y), rows, 1,
                                     N.PREC_FP32, N.ptr(self.ws), nbytes, st), "forward")
        for _ in range(2 if c["accumulate"] else 1):
            N.check(lib.b200_mlp_backward(C.byref(self.desc), N.ptr(self.flat), N.ptr(self.x), N.ptr(self.dy),
                                          N.ptr(self.dparams), N.ptr(self.dx), rows, N.PREC_FP32, N.ptr(self.ws),
                                          nbytes, st), "backward")
        torch.cuda.synchronize()

    def buf(self, off, cols):
        """rows x cols fp32 matrix at byte offset `off` from the workspace base."""
        rows = self.c["rows"]
        b = self.base + off
        return self.ws[b:b + rows * cols * 4].view(torch.float32).view(rows, cols)

    def act(self, l):
        if self.plan["act"][l] is None:
            return self.x
        return self.buf(self.plan["act"][l], self.plan["K"][l])

    def weight(self, l):
        k, n = self.plan["K"][l], self.plan["N"][l]
        return self.flat[self.w_off[l]:self.w_off[l] + k * n].view(n, k)

    def bias(self, l):
        return self.flat[self.b_off[l]:self.b_off[l] + self.plan["N"][l]]

    def dweight(self, l):
        k, n = self.plan["K"][l], self.plan["N"][l]
        return self.dparams[self.w_off[l]:self.w_off[l] + k * n].view(n, k)

    def dbias(self, l):
        return self.dparams[self.b_off[l]:self.b_off[l] + self.plan["N"][l]]


def _ratio(got, ref, bound):
    err = (got.double() - ref).abs()
    assert torch.isfinite(got).all(), "non-finite device value"
    r = torch.where(err == 0, torch.zeros_like(err), err / bound)
    return float(r.max()) if r.numel() else 0.0


def check_forward(run):
    c, pl = run.c, run.plan
    L, hid = c["layers"], c["hidden"]
    worst = {}
    if c["pe"]:
        b = _freqs(c["pe"]).to(DEV)
        arg = (run.x[:, :, None] * b[None, None, :]).double()          # the fp32 products the kernel forms
        ref = torch.cat((torch.sin(arg), torch.cos(arg)), dim=1).transpose(2, 1).reshape(c["rows"], -1)
        worst["encoding"] = _ratio(run.act(0), ref, 4 * U * ref.abs() + 2.0 ** -149)
        src = run.act(0)
    else:
        src = run.x
    for l in range(1, L):
        if pl["skip"][l]:
            assert torch.equal(run.act(l)[:, hid:], src), f"skip slot of layer {l} is not a copy of the layer-0 input"
    for l in range(L):
        a, w, b = run.act(l).double(), run.weight(l).double(), run.bias(l).double()
        z = a @ w.T + b
        bound = C_FP32 * U * math.sqrt(pl["K"][l]) * (a.abs() @ w.abs().T) + 4 * U * (b.abs() + z.abs())
        if l < L - 1:
            worst[f"act{l + 1}"] = _ratio(run.act(l + 1)[:, :hid], torch.relu(z), bound)
        else:
            ref = torch.tanh(z) if c["tanh"] else z
            worst["y"] = _ratio(run.y, ref, bound + (4 * U * ref.abs() if c["tanh"] else 0))
            assert torch.equal(run.buf(pl["y"], c["out_dim"]), run.y)
    return worst


def check_backward(run):
    c, pl = run.c, run.plan
    L, hid, rows = c["layers"], c["hidden"], c["rows"]
    times = 2.0 if c["accumulate"] else 1.0
    dy, y = run.dy.double(), run.y.double()
    if c["tanh"]:
        G, E = dy * (1 - y * y), 4 * U * dy.abs() * (1 + y * y)
    else:
        G, E = dy, torch.zeros_like(dy)
    acc = C_FP32 * U * (math.sqrt(min(rows, ROW_CHUNK)) + math.ceil(rows / ROW_CHUNK))
    worst = {}
    for l in range(L - 1, -1, -1):
        a = run.act(l).double()
        ga, aa = G.abs(), a.abs()
        worst[f"dW{l}"] = _ratio(run.dweight(l), times * (G.T @ a), times * (E.T @ aa + acc * (ga.T @ aa)))
        worst[f"db{l}"] = _ratio(run.dbias(l), times * G.sum(0), times * (E.sum(0) + acc * ga.sum(0)))
        w = run.weight(l).double()
        if l == 0:
            break
        wh = w[:, :hid]
        mask = (run.act(l)[:, :hid] > 0).double()
        E = mask * (E @ wh.abs() + C_FP32 * U * math.sqrt(pl["N"][l]) * (ga @ wh.abs()))
        G = mask * (G @ wh)
    # the last gradient buffer the device wrote holds G_0
    worst["dz0"] = _ratio(run.buf(pl["dz"][(L - 1) % 2], hid), G, E + 1e-300)
    d_in = G @ w
    e_in = E @ w.abs() + C_FP32 * U * math.sqrt(pl["N"][0]) * (G.abs() @ w.abs())
    if not c["pe"]:
        worst["dx"] = _ratio(run.dx, d_in, e_in + 1e-300)
        return worst
    worst["d_enc"] = _ratio(run.buf(pl["total"], pl["enc"]), d_in, e_in + 1e-300)
    F, d = c["pe"], c["in_dim"]
    sc = run.act(0).double().view(rows, F, 2, d)
    s, co = sc[:, :, 0], sc[:, :, 1]
    g4, e4 = d_in.view(rows, F, 2, d), e_in.view(rows, F, 2, d)
    ds, dc, es, ec = g4[:, :, 0], g4[:, :, 1], e4[:, :, 0], e4[:, :, 1]
    bk = _freqs(F).double().to(DEV)[None, :, None]
    ref = (bk * (ds * co - dc * s)).sum(1)
    bound = (bk * (es * co.abs() + ec * s.abs())).sum(1) + C_FP32 * U * (2 + F) * (bk * ((ds * co).abs() + (dc * s).abs())).sum(1)
    worst["dx"] = _ratio(run.dx, ref, bound + 1e-300)
    return worst


# ---------------------------------------------------------------------------------------------------------------
# CPU tests
# ---------------------------------------------------------------------------------------------------------------
def test_scratch_mirror_matches_workspace_bytes():
    """The mirror locates the device's intermediates: its total plus the 256-byte alignment slack is the library's
    workspace size for every case (none of them has tensor-core kernels, whose workspace is sized differently)."""
    lib = N.lib()
    for c in CASES.values():
        d = _desc(c)
        assert lib.b200_mlp_tc_architecture(C.byref(d)) == 0, c["name"]
        for rows in sorted({1, 127, 128, 129, c["rows"]}):
            assert plan(d, rows)["total"] + 256 == lib.b200_mlp_workspace_bytes(C.byref(d), rows, 1), (c["name"], rows)


def test_output_wider_than_hidden_sizes_gradient_buffers():
    """The output gradient is the first thing written into dz: the buffers are at least rows x out_dim."""
    lib = N.lib()
    for name in ("out3_hidden2", "out7_hidden2"):
        c = CASES[name]
        d = _desc(c)
        rp = _ceil128(c["rows"])
        pl = plan(d, c["rows"])
        assert pl["dz"][1] - pl["dz"][0] >= rp * c["out_dim"] * 4
        assert lib.b200_mlp_workspace_bytes(C.byref(d), c["rows"], 1) >= pl["dz"][1] + rp * c["out_dim"] * 4 + 256


def test_refused_shapes():
    from src.models.stage_1.implicit_neural_networks import IMLP
    # the reference's 0-wide encoding is a different network from "no encoding": refused, not rebuilt
    with pytest.raises(N.B200Error, match="positional_dim"):
        IMLP(3, 2, use_positional=True, positional_dim=0, verbose=False)
    IMLP(3, 2, use_positional=False, positional_dim=0, verbose=False)
    for key in ("positional_encoding_num_alpha", "positional_encoding_num_atlas"):
        with pytest.raises(N.B200Error, match=key):
            SG.seg_descs(dict(SG.SEG_DEFAULTS, **{key: 0}))
        with pytest.raises(N.B200Error, match=key):
            SG.SegTrainer(None, None, {key: 0}, device="cpu")
    for m in ("mapping1", "mapping2"):
        with pytest.raises(N.B200Error):
            SG.seg_descs(dict(SG.SEG_DEFAULTS, **{f"use_positional_encoding_{m}": True,
                                                   f"number_of_positional_encoding_{m}": 0}))
    assert SG.seg_descs(dict(SG.SEG_DEFAULTS, number_of_positional_encoding_mapping1=0))["mapping1"].pe_freqs == 0
    # depth 2..16 and at most 30 frequencies
    lib = N.lib()
    for layers, pe in ((1, 0), (17, 0), (4, 31), (4, -1)):
        d = A.make_desc(3, 2, 32, layers, pe, ())
        with pytest.raises(N.B200Error):
            A.mlp_layout(d)
        assert lib.b200_mlp_workspace_bytes(C.byref(d), 100, 1) == -1


# ---------------------------------------------------------------------------------------------------------------
# GPU: the case table
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_layer_by_layer_against_float64(name):
    run = Run(CASES[name])
    worst = check_forward(run)
    worst.update(check_backward(run))
    where = max(worst, key=worst.get)
    print(f"{name}: worst error / bound {worst[where]:.3f} ({where})")
    bad = {k: v for k, v in worst.items() if not v <= 1.0}
    assert not bad, (name, CASES[name]["branch"], bad)


@pytest.mark.gpu
def test_four_pe_skips_refused():
    """The encoding kernel writes at most three skip slots; a fourth is an error, not a silently missing copy."""
    d = A.make_desc(2, 2, 32, 8, 3, (1, 2, 3, 5))
    rows = 200
    nbytes = int(N.lib().b200_mlp_workspace_bytes(C.byref(d), rows, 1))
    ws = torch.zeros(nbytes, dtype=torch.uint8, device=DEV)
    _, _, total = A.mlp_layout(d)
    flat, x, y = torch.zeros(total, device=DEV), torch.zeros(rows, 2, device=DEV), torch.zeros(rows, 2, device=DEV)
    rc = N.lib().b200_mlp_forward(C.byref(d), N.ptr(flat), N.ptr(x), N.ptr(y), rows, 1, N.PREC_FP32, N.ptr(ws), nbytes,
                                  N.current_stream())
    assert rc != 0 and "skip" in N.last_error()
    torch.cuda.synchronize()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["pe10_in3", "pe_skip2", "skips_4_6", "hidden130", "out7_hidden2", "no_tanh_pe"])
def test_imlp_module_matches_c_abi(name):
    """The `IMLP` class sizes its own workspace (including the encoded-input gradient of a PE network): with x
    requiring grad its output and gradients are bit-identical to the checked C-ABI call (<= 1024 rows: one
    weight-gradient chunk, so one atomic per gradient and a deterministic result)."""
    from src.models.stage_1.implicit_neural_networks import IMLP
    c = CASES[name]
    assert c["rows"] <= ROW_CHUNK
    run = Run(c)
    assert max(check_forward(run).values()) <= 1.0 and max(check_backward(run).values()) <= 1.0
    net = IMLP(c["in_dim"], c["out_dim"], c["hidden"], use_positional=c["pe"] > 0, positional_dim=max(c["pe"], 1),
               skip_layers=list(c["skips"]), num_layers=c["layers"], verbose=False, use_tanh=c["tanh"]).to(DEV)
    with torch.no_grad():
        net.flat.copy_(run.flat)
    x = run.x.detach().clone().requires_grad_(True)
    y = net(x)
    y.backward(run.dy)
    torch.cuda.synchronize()
    assert torch.equal(y.detach(), run.y)
    assert torch.equal(net.flat.grad, run.dparams)
    assert torch.equal(x.grad, run.dx)


# ---------------------------------------------------------------------------------------------------------------
# GPU: the segmentation trip with networks that have no tensor-core kernels
# ---------------------------------------------------------------------------------------------------------------
# mapping1 keeps its default (tensor cores at B200_PREC_TC); the other three leave them
MIXED = dict(number_of_channels_mapping2=128, number_of_layers_alpha=6, positional_encoding_num_atlas=6)
MIXED_ARCH = dict(mapping1=1, mapping2=0, alpha=0, atlas=0)


def _mixed_specs():
    return dict(mapping1=S.MAPPING1_SPEC, mapping2=O.MlpSpec(3, 2, 128, False, 2, (), 4),
                alpha=O.MlpSpec(3, 1, 256, True, 5, (), 6), atlas=O.MlpSpec(2, 3, 256, True, 6, (4, 7), 8))


def _seg_setup(golden_dir, specs):
    """The fixture's video, matte and index batch, with networks of `specs` drawn from the fixture's seed."""
    z, video, masks, _ = load_fixture(golden_dir)
    torch.manual_seed(int(z["init_seed"]))
    return z, video, masks, S.init_nets(specs)


def _seg_trainer(video, masks, nets, config, precision, batch, t0=0, t1=None):
    data = dict(frames=video.frames, frames_dx=video.frames_dx, frames_dy=video.frames_dy, flow_fwd=video.flow_fwd,
                flow_bwd=video.flow_bwd, mask_fwd=video.mask_fwd, mask_bwd=video.mask_bwd)
    vid = A.DeviceVideo.from_reference_layout(data, DEV, t0, t1)
    tr = SG.SegTrainer(vid, SG.pack_mask_frames(masks, DEV, t0, t1), dict(config, samples_batch=batch),
                       precision=precision, device=DEV)
    tr.load_state({k: O.state_dict_of(nets[k]) for k in ORDER})
    return tr


def _need_tc():
    if not N.lib().b200_device_supports_tc():
        pytest.skip("no sm_90 device")


def _check_trip(losses, grad_views, video, masks, nets, specs, inds, it, tc, label):
    """Losses and gradients against the oracle with the bounds of tests/test_seg_gpu.py for the precision."""
    mine = {k: [p.clone().requires_grad_(True) for p in nets[k]] for k in ORDER}
    terms = S.seg_iteration_losses(video, masks, mine, inds, it, specs=specs)
    terms["total"].backward()
    for k, v in terms.items():
        np.testing.assert_allclose(losses[k], float(v.detach()), rtol=2e-3 if tc else 2e-4, err_msg=k)
    worst = 0.0
    for k in ORDER:
        scale_net = max(float(p.grad.abs().max()) for p in mine[k])
        for (name, g), p in zip(grad_views(k).items(), mine[k]):
            bound = (1.5e-2 if tc else 1e-3) * float(p.grad.abs().max()) + (2e-3 if tc else 2e-4) * scale_net + 1e-7
            err = float((g.detach().cpu().double() - p.grad.double()).abs().max())
            worst = max(worst, err / bound)
            assert err <= bound, (label, k, name, err, bound)
    print(f"{label}: worst gradient error / bound {worst:.3f}")


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["mixed", "fp32"])
@pytest.mark.parametrize("it", [0, 6000])
def test_seg_trip_with_fp32_networks(golden_dir, mode, it):
    """One trip with mapping2 128 wide, a 6-layer alpha and a 6-frequency atlas: at B200_PREC_TC only mapping1 runs
    on the tensor cores (tensor-core bounds), at B200_PREC_FP32 none does (fp32 bounds)."""
    if mode == "mixed":
        _need_tc()
    specs = _mixed_specs()
    z, video, masks, nets = _seg_setup(golden_dir, specs)
    inds = torch.from_numpy(z["inds"])
    tr = _seg_trainer(video, masks, nets, MIXED, N.PREC_TC if mode == "mixed" else N.PREC_FP32, inds.shape[0])
    for k, arch in MIXED_ARCH.items():
        assert N.lib().b200_mlp_tc_architecture(C.byref(tr.descs[k])) == arch, k
    tr.indices.copy_(inds.reshape(-1))
    tr.loss_grad(it)
    torch.cuda.synchronize()
    _check_trip(tr.loss_dict(), tr.grad_views, video, masks, nets, specs, inds, it, mode == "mixed", f"seg {mode} it {it}")


@pytest.mark.gpu
def test_seg_mixed_trip_two_shard_sum(golden_dir):
    """2-way frame split of the mixed trip, the shards evaluated one after the other.  The fp32 networks evaluate every
    row of the batch, padding slots and dead compacted flow rows included: the sum is right only if the loss head
    writes zero gradients for those rows."""
    from test_seg_sharding_gloo import global_flow_counts
    _need_tc()
    specs = _mixed_specs()
    z, video, masks, nets = _seg_setup(golden_dir, specs)
    inds = torch.from_numpy(z["inds"])
    total, world = None, 2
    for r in range(world):
        t0, t1 = A.frame_range(r, world, video.T)
        tr = _seg_trainer(video, masks, nets, MIXED, N.PREC_TC, inds.shape[0], t0, t1)
        tr.indices.copy_(inds.reshape(-1))
        tr.loss_grad(0)
        torch.cuda.synchronize()
        part = tr.grad_loss.detach().cpu().double()
        total = part if total is None else total + part
    losses = {k: float(v) for k, v in zip(SG.LOSS_NAMES, total[tr.n_params:])}
    n_f, n_b = global_flow_counts(video, inds)
    assert (losses["n_fwd"], losses["n_bwd"]) == (world * n_f, world * n_b)
    grads = total[:tr.n_params].float()
    _check_trip(losses, lambda k: tr._views(grads, k), video, masks, nets, specs, inds, 0, True, "seg mixed 2-way shard sum")


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["mixed", "fp32"])
def test_seg_render_with_fp32_networks(golden_dir, mode):
    """Reconstruction and alpha of the mixed configuration against the oracle's render, to 2e-5 (the bound of
    test_seg_gpu's fp32 render) in both modes: alpha comes from an fp32 network either way, and mapping1's fp32-grade
    tensor-core forward stays within it (measured 1.8e-7 on an H100 80GB HBM3 at 400 W)."""
    if mode == "mixed":
        _need_tc()
    specs = _mixed_specs()
    z, video, masks, nets = _seg_setup(golden_dir, specs)
    tr = _seg_trainer(video, masks, nets, MIXED, N.PREC_TC if mode == "mixed" else N.PREC_FP32, 64)
    img, alpha = tr.render_frame(2, video.H, video.W, video.T, chunk=500)
    ref_img, ref_alpha = S.render_frame_seg(nets, 2, video.H, video.W, video.T, specs=specs)
    e_img = float((img.cpu() - ref_img).abs().max())
    e_alpha = float((alpha.cpu() - ref_alpha).abs().max())
    print(f"seg render {mode}: max |img - ref| {e_img:.2e}, max |alpha - ref| {e_alpha:.2e}")
    assert e_alpha <= 2e-5
    assert e_img <= 2e-5


@pytest.mark.gpu
def test_seg_pretrain_64_channel_mapping(golden_dir):
    """pre_train_mapping of a 64-channel mapping1 (no tensor-core kernels: the trainer's B200_PREC_TC falls back to
    fp32 for it) against the oracle loop of test_seg_gpu's pre-training test, with its fp32 bounds."""
    specs = dict(_mixed_specs(), mapping1=O.MlpSpec(3, 2, 64, False, 4, (), 6))
    config = dict(MIXED, number_of_channels_mapping1=64)
    z, video, masks, nets = _seg_setup(golden_dir, specs)
    prec = N.PREC_TC if N.lib().b200_device_supports_tc() else N.PREC_FP32
    tr = _seg_trainer(video, masks, nets, config, prec, 64)
    assert N.lib().b200_mlp_tc_architecture(C.byref(tr.descs["mapping1"])) == 0
    Hp, Wp, Tp = 20, 36, 2
    mp = [p.clone().requires_grad_(True) for p in nets["mapping1"]]
    opt = torch.optim.Adam(mp, lr=1e-4)
    torch.manual_seed(5)
    want = []
    for f in range(Tp):
        ys = torch.randint(Hp, (10000, 1)); xs = torch.randint(Wp, (10000, 1))
        i_s, j_s = ys / O._half(max(Wp, Hp)) - 1, xs / O._half(max(Wp, Hp)) - 1
        xyt = torch.cat((j_s, i_s, (f / (Tp / 2.0) - 1) * torch.ones_like(i_s)), dim=1)
        loss = (xyt[:, :2] * 0.8 - O.mlp_forward(specs["mapping1"], mp, xyt)).norm(dim=1).mean()
        opt.zero_grad(); loss.backward(); opt.step()
        want.append(float(loss.detach()))
    torch.manual_seed(5)
    last = tr.pretrain("mapping1", Tp, Hp, Wp, 1)
    np.testing.assert_allclose(float(last), want[-1], rtol=2e-4)
    for (name, v), p in zip(tr.param_views("mapping1").items(), mp):
        np.testing.assert_allclose(v.cpu().numpy(), p.detach().numpy(), rtol=0, atol=5e-5, err_msg=name)
