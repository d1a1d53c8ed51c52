"""The ConvLSTM with a carried state: the fused gate layer (b200_convlstm_tma: gate convolution on wgmma with the cell
update in its epilogue), the fp32 cell kernel (b200_convlstm_cell) and TransformNet's recurrence.

Fused layer, one layer at a time, against float64 on the operands the kernel rounds (saturate, then RN to fp16, as
in test_conv_kernels_gpu.py).  Each gate z obeys the convolution bound of that file,
    E_z = c * u * sqrt(R) * A + 4u * |z|         (u = 2^-24, R = Cin * 9, A = conv64(|x16|, |w16|) + |b|, c = 4),
and the bound is carried through the cell with sigma' <= 1/4, tanh' <= 1 and 8u * |value| for each expf / tanhf
based function (a few ulps):
    E_sig = E_z / 4 + 8u |sig|,   E_tanh = E_z + 8u |tanh|
    E_cell = |c_prev| E_rem + |g| E_in + |in| E_g + E_in E_g + 4u (|rem c_prev| + |in g|)
    E_hidden = |tanh(cell)| E_out + |out| (E_cell + 8u |tanh(cell)|) + E_out E_cell + 4u |hidden|
Every case prints the largest err / bound it measured and names the planner branch it lands in (n_tile, N tiles,
folded x taps), checked against the planner mirror of test_conv_kernels_gpu.py.

With prev_cell = NULL the fused layer is bit-identical to the gate convolution followed by
b200_convlstm_zero_state, and with a state to the gate convolution on cat(x, prev_hidden) followed by
b200_convlstm_cell: the same fp16 operands, the same MMAs per gate column (the interleaving only permutes columns)
and the same cell expressions."""
import ctypes as C
import math
import os
import types

import pytest
import torch
import torch.nn.functional as F

from b200 import _native as N
from b200 import nn as K
from convlstm_state_common import recurrence, recurrence_inputs, transformnet_forward_state
from csrc_build import ensure_built
from nets_common import seeded_weights
from conv_common import cell_reference, convlstm_reference
from test_conv_kernels_gpu import plan, spec

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture(scope="module", autouse=True)
def _built():
    ensure_built()


# name -> (C, n, h, w, chained, with prev_cell, want_cell, planner fields of the gate layer)
CASES = {
    "c16_zero": (16, 1, 9, 40, False, False, True, dict(n_tile=64, n_tiles_n=1, fold_cf=16)),
    "c16_state": (16, 1, 9, 40, False, True, True, dict(n_tile=64, n_tiles_n=1, fold_cf=0)),
    "c16_state_chained": (16, 1, 9, 40, True, True, True, dict(n_tile=64, n_tiles_n=1, fold_cf=0)),
    "c32_zero_chained": (32, 1, 7, 33, True, False, True, dict(n_tile=128, n_tiles_n=1, fold_cf=0)),
    "c32_state_nocell": (32, 1, 7, 33, False, True, False, dict(n_tile=128, n_tiles_n=1, fold_cf=0)),
    "c64_state_n2": (64, 2, 6, 50, False, True, True, dict(n_tile=256, n_tiles_n=1, fold_cf=0)),
    "c64_zero_n2_chained": (64, 2, 6, 50, True, False, True, dict(n_tile=256, n_tiles_n=1, fold_cf=0)),
    "c128_state_w150": (128, 1, 5, 150, False, True, True, dict(n_tile=256, n_tiles_n=2, x_tiles=2)),
    "c128_state_w150_chained": (128, 1, 5, 150, True, True, True, dict(n_tile=256, n_tiles_n=2, x_tiles=2)),
    "c128_zero_nocell_chained": (128, 2, 5, 150, True, False, False, dict(n_tile=256, n_tiles_n=2, x_tiles=2)),
}


def _case_inputs(name, c, n, h, w, scale=3.0):
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    x = torch.randn(n, c, h, w, generator=g)
    wt = torch.randn(4 * c, 2 * c, 3, 3, generator=g) / math.sqrt(2 * c * 9) * 2.0
    b = torch.randn(4 * c, generator=g)
    h0 = (torch.rand(n, c, h, w, generator=g) * 2 - 1) * scale
    c0 = torch.randn(n, c, h, w, generator=g) * scale
    return x, wt, b, h0, c0


def _pack(chain, t, c_off):
    N.check(N.lib().b200_conv_tma_pack_chain(C.byref(chain.desc), N.ptr(t), t.shape[1], N.ptr(chain.buf), c_off,
                                             N.current_stream()), "b200_conv_tma_pack_chain")


def _run_fused(name, x, wt, b, state, chained, want_cell):
    """K.convlstm on the device: unchained (tensor input) or chained (x packed into a Chain of C or 2C channels)."""
    n, c, h, w = x.shape
    xd, bd = x.to(DEV), b.to(DEV)
    wd = wt.to(DEV) if state is not None else wt[:, :c].contiguous().to(DEV)
    sd = None if state is None else tuple(t.to(DEV) for t in state)
    if chained:
        ch = K.Chain(n, 2 * c if state is not None else c, h, w, (3, 3), 1, DEV, tag=f"test_convlstm_{name}")
        _pack(ch, xd, 0)
        xd = ch
    return K.convlstm(xd, wd, bd, sd, want_cell=want_cell)


def _reference(x, wt, b, state):
    """float64 (hidden, cell) on the kernel's fp16 operands, and their elementwise bounds (module docstring)."""
    c = x.shape[1]
    if state is None:
        return convlstm_reference(x, wt[:, :c], b, None)
    return convlstm_reference(torch.cat((x, state[0]), 1), wt, b, state[1])


def _gate_case(c, n, h, w, state):
    cin = 2 * c if state else c
    return spec("gates", n=n, cin=cin, h=h, w=w, cout=4 * c)


@pytest.mark.parametrize("name", list(CASES))
def test_fused_layer_against_float64(name):
    c, n, h, w, chained, with_prev, want_cell, expect = CASES[name]
    p = plan(_gate_case(c, n, h, w, with_prev))
    for key, val in expect.items():
        assert p[key] == val, (name, key, p[key], val)
    x, wt, b, h0, c0 = _case_inputs(name, c, n, h, w)
    state = (h0, c0) if with_prev else None
    hid, cell = _run_fused(name, x, wt, b, state, chained, want_cell)
    assert (cell is None) == (not want_cell)
    ref_h, ref_c, e_h, e_c = _reference(x, wt, b, state)
    ratios = {}
    for what, got, ref, e in (("hidden", hid, ref_h, e_h), ("cell", cell, ref_c, e_c)):
        if got is None:
            continue
        got = got.cpu().double()
        assert got.shape == ref.shape and torch.isfinite(got).all(), what
        err = (got - ref).abs()
        ratios[what] = float((err / e.clamp_min(1e-300)).max())
        assert bool((err <= e).all()), f"{name} {what}: {int((err > e).sum())} elements beyond the bound"
    print(f"{name}: err / bound = " + ", ".join(f"{k} {v:.3f}" for k, v in ratios.items()))


@pytest.mark.parametrize("chained", [False, True])
@pytest.mark.parametrize("c", [32, 128])
def test_fused_zero_state_equals_conv_then_cell(c, chained):
    """prev_cell NULL: the fused layer equals b200_conv2d_tma_chain's gates followed by b200_convlstm_zero_state."""
    n, h, w = 1, 11, 140
    x, wt, b, _, _ = _case_inputs(f"bitwise{c}", c, n, h, w)
    w_in = wt[:, :c].contiguous().to(DEV)
    xd, bd = x.to(DEV), b.to(DEV)
    src = xd
    if chained:
        src = K.Chain(n, c, h, w, (3, 3), 1, DEV, tag="test_convlstm_bitwise")
        _pack(src, xd, 0)
    gates = K.conv2d(src, w_in, bd, pad=1, precision="tc")
    h_ref, c_ref = K.convlstm_zero_state(gates)
    hid, cell = K.convlstm(src, w_in, bd)
    assert torch.equal(hid, h_ref) and torch.equal(cell, c_ref)


@pytest.mark.parametrize("chained", [False, True])
def test_fused_state_equals_conv_then_cell(chained):
    """With a state: the fused layer equals the gate convolution on cat(x, prev_hidden) followed by b200_convlstm_cell
    (the chained input packs prev_hidden with b200_conv_tma_pack_chain, the unchained one repacks the concatenation)."""
    c, n, h, w = 128, 2, 6, 131
    x, wt, b, h0, c0 = _case_inputs("bitwise_state", c, n, h, w)
    xd, wd, bd, hd, cd = (t.to(DEV) for t in (x, wt, b, h0, c0))
    gates = K.conv2d(torch.cat((xd, hd), 1), wd, bd, pad=1, precision="tc")
    h_ref, c_ref = K.convlstm_cell(gates, cd)
    src = xd
    if chained:
        src = K.Chain(n, 2 * c, h, w, (3, 3), 1, DEV, tag="test_convlstm_bitwise_state")
        _pack(src, xd, 0)
    hid, cell = K.convlstm(src, wd, bd, (hd, cd))
    assert torch.equal(hid, h_ref) and torch.equal(cell, c_ref)


@pytest.mark.parametrize("with_prev", [False, True])
def test_fp32_cell_kernel_against_float64(with_prev):
    """b200_convlstm_cell on fp32 gates: a few ulps of float64 (the bound of the module docstring with E_z = 0)."""
    g = torch.Generator().manual_seed(61)
    n, c, h, w = 2, 24, 7, 19
    gates = torch.randn(n, 4 * c, h, w, generator=g) * 4
    prev = torch.randn(n, c, h, w, generator=g) * 3 if with_prev else None
    hid, cell = K.convlstm_cell(gates.to(DEV), None if prev is None else prev.to(DEV))
    ref_h, ref_c, e_h, e_c = cell_reference(gates.double(), torch.zeros_like(gates.double()), prev)
    for what, got, ref, e in (("cell", cell, ref_c, e_c), ("hidden", hid, ref_h, e_h)):
        err = (got.cpu().double() - ref).abs()
        print(f"fp32 cell prev={with_prev} {what}: err / bound = {float((err / e.clamp_min(1e-300)).max()):.3f}")
        assert bool((err <= e).all()), what


def _transformnet(fx):
    from src.models.network_local import TransformNet
    tn = TransformNet(types.SimpleNamespace(nf=fx["nf"], norm="IN", model="TransformNet", blocks=5), nc_in=12, nc_out=3)
    sd = seeded_weights(fx["shapes"], fx["seed"])
    tn.load_state_dict(sd, strict=False)
    return tn.to(DEV), sd


def _rel(a, b):
    return ((a.cpu() - b).abs().max() / b.abs().max()).item()


@pytest.mark.parametrize("prec", ["fp32", "tc"])
def test_transformnet_recurrence_against_the_reference(golden_dir, prec):
    """The fixture's 4-frame recurrence (each call fed the state the previous call returned) and its random-state
    step, against the CPU restatement that test_convlstm_state_cpu.py pins to the reference's outputs: fp32
    convolutions within 1e-4 absolute, wgmma convolutions within 2e-2 * max|output| per frame."""
    fx = torch.load(os.path.join(golden_dir, "transformnet_state.pt"))
    tn, sd = _transformnet(fx)
    xs, x_r, state_r = recurrence_inputs(fx["input_seed"], nf=fx["nf"])
    with torch.no_grad():
        ref_ys, ref_state = recurrence(sd, xs)
        ref_r = transformnet_forward_state(sd, x_r, state_r)
    prev = K.set_conv_precision(prec)
    try:
        state, outs = None, []
        for x in xs:
            y, state = tn(x.to(DEV), state)
            outs.append(y)
        r_y, (r_h, r_c) = tn(x_r.to(DEV), tuple(t.to(DEV) for t in state_r))
    finally:
        K.set_conv_precision(prev)
    pairs = [(f"Y{t}", y, ref_ys[t]) for t, y in enumerate(outs)]
    pairs += [("hidden", state[0], ref_state[0]), ("cell", state[1], ref_state[1]), ("r_Y", r_y, ref_r[0]),
              ("r_hidden", r_h, ref_r[1]), ("r_cell", r_c, ref_r[2])]
    if prec == "fp32":
        errs = {k: (a.cpu() - b).abs().max().item() for k, a, b in pairs}
        print("TransformNet recurrence [fp32] abs:", {k: f"{v:.2e}" for k, v in errs.items()})
        assert max(errs.values()) <= 1e-4, errs
    else:
        errs = {k: _rel(a, b) for k, a, b in pairs}
        print("TransformNet recurrence [tc] rel:", {k: f"{v:.2e}" for k, v in errs.items()})
        assert max(errs.values()) <= 2e-2, errs


def test_returned_state_is_fresh_and_reusable(golden_dir):
    """The returned state is new tensors, never cached buffers: feeding it back leaves it unchanged, and a second
    network call does not overwrite the first call's outputs."""
    fx = torch.load(os.path.join(golden_dir, "transformnet_state.pt"))
    tn, _ = _transformnet(fx)
    xs, _, _ = recurrence_inputs(fx["input_seed"], nf=fx["nf"])
    prev = K.set_conv_precision("tc")
    try:
        y1, s1 = tn(xs[0].to(DEV), None)
        keep = [t.clone() for t in (y1, *s1)]
        y2, s2 = tn(xs[1].to(DEV), s1)
        y3, s3 = tn(xs[1].to(DEV), s1)
    finally:
        K.set_conv_precision(prev)
    assert all(torch.equal(a, b) for a, b in zip(keep, (y1, *s1)))
    assert torch.equal(y2, y3) and torch.equal(s2[0], s3[0]) and torch.equal(s2[1], s3[1])
    assert len({t.data_ptr() for t in (*s1, *s2, *s3)}) == 6


def test_stateful_transformnet_1088x1920_tensor_cores(golden_dir):
    """One stateful step at the benchmark's size against the oracle: 5e-3 * max|output| as in test_nets_fullsize_gpu."""
    fx = torch.load(os.path.join(golden_dir, "transformnet_state.pt"))
    tn, sd = _transformnet(fx)
    hp, wp = 1088, 1920
    g = torch.Generator().manual_seed(71)
    x = F.interpolate(torch.rand(1, 12, hp // 16, wp // 16, generator=g), size=(hp, wp), mode="bilinear",
                      align_corners=False).contiguous()
    c = 4 * fx["nf"]
    h0 = torch.tanh(torch.randn(1, c, hp // 4, wp // 4, generator=g))
    c0 = torch.randn(1, c, hp // 4, wp // 4, generator=g)
    with torch.no_grad():
        oy, oh, oc = transformnet_forward_state(sd, x, (h0, c0))
    prev = K.set_conv_precision("tc")
    try:
        y, (hid, cell) = tn(x.to(DEV), (h0.to(DEV), c0.to(DEV)))
    finally:
        K.set_conv_precision(prev)
    errs = {"Y": _rel(y, oy), "hidden": _rel(hid, oh), "cell": _rel(cell, oc)}
    print("stateful TransformNet at 1088x1920 [tc]:", errs)
    assert max(errs.values()) <= 5e-3, errs


@pytest.mark.parametrize("bad", ["shape", "device", "noncontig", "dtype", "not_a_pair"])
def test_bad_states_are_refused(bad):
    c, n, h, w = 32, 1, 6, 20
    x, wt, b, h0, c0 = _case_inputs("refuse", c, n, h, w)
    xd, wd, bd = x.to(DEV), wt.to(DEV), b.to(DEV)
    hd, cd = h0.to(DEV), c0.to(DEV)
    state = {"shape": (hd[:, :, :5].contiguous(), cd),
             "device": (hd, c0),
             "noncontig": (hd, torch.empty(n, c, w, h, device=DEV).transpose(2, 3)),
             "dtype": (hd.double(), cd),
             "not_a_pair": (hd,)}[bad]
    with pytest.raises(N.B200Error):
        K.convlstm(xd, wd, bd, state)
    prev = K.set_conv_precision("fp32")
    try:
        from src.models.network_local import ConvLSTM
        m = ConvLSTM(c, c, 3).to(DEV)
        with pytest.raises(N.B200Error):
            m.run(xd, state)
    finally:
        K.set_conv_precision(prev)
