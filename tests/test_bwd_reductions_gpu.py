"""Bias gradients of every layer and the plain mapping's first-layer weight gradient dW0 from the fused tensor-core
backward (tc_bwd_kernel), all six networks, against float64.

tc_bwd_kernel forms these sums with m64n8k16 MMAs over each dZ tile it has written in shared memory: the tile's two
fp16 terms (hi + lo of S_g * dZ, 22 significand bits) against a [1, 0, x_hi, x_lo, y_hi, y_lo, t_hi, t_lo] operand.

Bound per column n of a layer i, with A = the float64 sum over rows of the absolute-value chain (|dZ| propagated
through |W| with the reference's ReLU masks; |dZ0|^T |x| for dW0), u = 2^-22 the 2-term split's relative precision:
    |g - g64| <= u (4 (L - 1 - i) + 4) A                  each dgrad layer below the output: split dZ, split W, the
                                                          dropped lo*lo term, one more for the fp32 products
               + 2^-24 (64 + tiles per CTA + CTAs) A      one fp32 rounding per addition along the longest chain: the
                                                          tile's 64 rows in the MMA, the CTA's tiles in shared memory,
                                                          one global atomic per CTA
               + flip slack                               (first order) what a ReLU mask that the kernel's fp32-grade
                                                          forward may set differently could change: every
                                                          pre-activation within 2^-15 of its |W||h| + |b| scale, its
                                                          unmasked gradient propagated down through |W|, plus u |dy|
                                                          (tanh' of the kernel's own output, evaluated in fp32)
                                                          propagated the same way
dW0 adds u for the split of x.  The output layer's bias b_{L-1} is an fp32 warp sum per tile and one global atomic per
warp: 2^-24 (8 + 8 tiles) A.

Cases: one partial tile (77 rows, 131 of 132 CTAs have no tile), many tiles per CTA with a ragged last tile, and the
stage-1 step itself, whose mapping runs on nine row groups with the two flow-match groups compacted to their valid rows
(ragged last tiles inside the batch).  Each prints the largest ratio of error to bound.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from b200 import _native as N
from b200 import atlas as A
from b200 import synth
from oracle import atlas_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda"
U22 = 2.0 ** -22
U24 = 2.0 ** -24
FLIP = 2.0 ** -15
SMS = 132

# (IMLP ctor arguments, oracle spec, input scale / shift) of the six networks with a tensor-core backward
NETS = {
    "mapping": (dict(input_dim=3, output_dim=2, use_positional=False, positional_dim=4, num_layers=6, skip_layers=[]),
                O.MlpSpec(3, 2, 256, False, 4, (), 6), 2.0, -1.0),
    "mapping4": (dict(input_dim=3, output_dim=2, use_positional=False, positional_dim=2, num_layers=4, skip_layers=[]),
                 O.MlpSpec(3, 2, 256, False, 2, (), 4), 2.0, -1.0),
    "atlas": (dict(input_dim=2, output_dim=3, use_positional=True, positional_dim=10, num_layers=8, skip_layers=[4, 7]),
              O.ATLAS_SPEC, 1.0, 0.0),
    "alpha": (dict(input_dim=3, output_dim=1, use_positional=True, positional_dim=5, num_layers=8, skip_layers=[]),
              O.MlpSpec(3, 1, 256, True, 5, (), 8), 2.0, -1.0),
    "pe6": (dict(input_dim=3, output_dim=2, use_positional=True, positional_dim=4, num_layers=6, skip_layers=[]),
            O.MlpSpec(3, 2, 256, True, 4, (), 6), 2.0, -1.0),
    "pe4": (dict(input_dim=3, output_dim=2, use_positional=True, positional_dim=10, num_layers=4, skip_layers=[]),
            O.MlpSpec(3, 2, 256, True, 10, (), 4), 2.0, -1.0),
}


def _need_tc():
    if not N.lib().b200_device_supports_tc():
        pytest.skip("no sm_90 device")


def reference(spec, params, x, dy, y_dev):
    """float64 bias gradients of every layer and dW0, with the absolute-value chain A and the flip slack of each.
    tanh' is taken of the kernel's own output y_dev, as the kernel does (its fp32 evaluation: slack 2^-22 |dy|), and
    the encoding of the fp32 products x b_k, as the kernel forms them (the float64 products would move the arguments of
    the 2^9 pi frequency by up to 1e-4)."""
    p = [t.double() for t in params]
    L = spec.num_layers
    if spec.use_positional:
        arg = (x.float()[:, :, None] * O.pe_frequencies(spec).float()[None, None, :]).double()
        enc = torch.cat((torch.sin(arg), torch.cos(arg)), dim=1).transpose(2, 1).reshape(x.shape[0], -1)
    else:
        enc = x.double()
    z, scale = [], []
    for i in range(L):
        inp = enc if i == 0 else torch.relu(z[-1])
        ainp = inp.abs()
        if i > 0 and i in spec.skip_layers:
            inp = torch.cat((inp, enc), 1)
            ainp = torch.cat((ainp, enc.abs()), 1)
        z.append(inp @ p[2 * i].T + p[2 * i + 1])
        scale.append(ainp @ p[2 * i].abs().T + p[2 * i + 1].abs())
    y = y_dev.double()
    dz = dy.double() * ((1 - y * y) if spec.use_tanh else 1.0)
    adz = dz.abs()
    slack = U22 * dy.double().abs()
    out = {}
    for i in range(L - 1, -1, -1):
        out[i] = (dz.sum(0), adz.sum(0), slack.sum(0))
        if i == 0:
            out["w0"] = (dz.T @ enc, adz.T @ enc.abs(), slack.T @ enc.abs())
            break
        w = p[2 * i][:, :spec.hidden_dim]
        dh, adh, sh = dz @ w, adz @ w.abs(), slack @ w.abs()
        mask = (z[i - 1] > 0).double()
        near = (z[i - 1].abs() <= FLIP * scale[i - 1]).double()
        dz, adz, slack = dh * mask, adh * mask, sh + dh.abs() * near
    return out


def check(spec, got_bias, got_w0, ref, tiles, label):
    """got_bias[i]: device bias gradient of layer i; got_w0: device dW0 (plain mapping) or None.  Returns the largest
    ratio of error to bound."""
    L = spec.num_layers
    acc = U24 * (64 + (tiles + SMS - 1) // SMS + min(SMS, tiles))
    worst = 0.0
    problems = []
    items = [(i, got_bias[i], ref[i], U22 * (4 * (L - 1 - i) + 4) + acc) for i in range(L - 1)]
    items.append((L - 1, got_bias[L - 1], ref[L - 1], U24 * (8 + 8 * tiles)))
    if got_w0 is not None:
        items.append(("w0", got_w0, ref["w0"], U22 * (4 * (L - 1) + 5) + acc))
    for key, got, (g64, a64, s64), coef in items:
        err = (got.double().cpu() - g64).abs()
        bound = coef * a64 + s64 + 1e-30
        ratio = float((err / bound).max())
        worst = max(worst, ratio)
        if ratio > 1.0:
            problems.append((label, key, ratio, float(err.max())))
    assert not problems, problems
    return worst


@pytest.mark.parametrize("rows", [77, 3 * SMS * 128 - 50])
@pytest.mark.parametrize("which", sorted(NETS))
def test_bias_and_dw0_row_sums(which, rows, monkeypatch):
    _need_tc()
    monkeypatch.setenv("B200_IMLP_PRECISION", "tc")
    from src.models.stage_1.implicit_neural_networks import IMLP
    kw, spec, xs, xo = NETS[which]
    net = IMLP(hidden_dim=256, verbose=False, **kw)
    assert net._tc_arch in (1, 2, 3, 4)
    torch.manual_seed(1000 + rows + len(which))
    params = O.init_mlp(spec)
    net.load_state_dict(O.state_dict_of(params))
    net = net.to(DEV)
    g = torch.Generator().manual_seed(rows)
    x = torch.rand(rows, spec.input_dim, generator=g) * xs + xo
    dy = torch.randn(rows, spec.output_dim, generator=g)
    y = net(x.to(DEV))
    y.backward(dy.to(DEV))
    torch.cuda.synchronize()
    views = net._views(net.flat.grad)
    L = spec.num_layers
    got_bias = [views[f"hidden.{i}.bias"] for i in range(L)]
    got_w0 = views["hidden.0.weight"] if not spec.use_positional else None
    worst = check(spec, got_bias, got_w0, reference(spec, params, x, dy, y.detach().cpu()), (rows + 127) // 128, which)
    print(f"{which} rows {rows}: largest |err| / bound {worst:.3g}")


def test_mapping_row_sums_compacted_groups(golden_dir):
    """The stage-1 step's mapping backward: nine groups, the flow-match groups compacted (ragged last tiles)."""
    _need_tc()
    H, W, T, B = 24, 40, 6, 300
    data = synth.throughput_set(H, W, T, seed=3)
    z = np.load(f"{golden_dir}/params_seed1234.npz")
    mp = [torch.from_numpy(z[f"map{i}"]) for i in range(12)]
    ap = [torch.from_numpy(z[f"atl{i}"]) for i in range(16)]
    vid = A.DeviceVideo.from_reference_layout(data, DEV)
    tr = A.AtlasTrainer(vid, {"samples_batch": B}, precision=N.PREC_TC, device=DEV)
    tr.load_state(O.state_dict_of(mp), O.state_dict_of(ap))
    tr.indices.copy_(torch.randint(H * W * T, (B,), generator=torch.Generator().manual_seed(2)))
    tr.loss_grad(True)
    torch.cuda.synchronize()
    view = tr.workspace_views()
    cap = view["cap"]
    cfg = tr._config(True)
    ws = tr._workspace()
    off = (C.c_int64 * 8)()
    N.check(N.lib().b200_atlas_workspace_offsets_for(C.byref(cfg), C.byref(tr.map_desc), N.ptr(ws), off), "offsets")
    d_uv = ws[off[4]:off[4] + 4 * 9 * cap * 2].view(torch.float32).view(9 * cap, 2).cpu()
    x = view["x_map"].reshape(9 * cap, 4).cpu()[:, :3]
    uv = view["uv"].reshape(9 * cap, 2).cpu()
    cnt = view["counters"].cpu()
    live = torch.zeros(9 * cap, dtype=torch.bool)
    ragged = tiles = 0
    for grp in range(9):
        n = int(cnt[grp]) if grp in (5, 6) else B
        live[grp * cap:grp * cap + n] = True
        ragged += n % 128 != 0
        tiles += (n + 127) // 128
    assert int(cnt[5]) < B and int(cnt[6]) < B and ragged >= 2
    views = tr._views(tr.grads, "mapping")
    spec = O.MAPPING_SPEC
    got_bias = [views[f"hidden.{i}.bias"] for i in range(spec.num_layers)]
    rows = int(live.sum())
    worst = check(spec, got_bias, views["hidden.0.weight"], reference(spec, mp, x[live], d_uv[live], uv[live]), tiles,
                  "step")
    print(f"stage-1 step mapping, {rows} live rows: largest |err| / bound {worst:.3g}")
