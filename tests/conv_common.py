"""Operand-exact float64 references of the convolution layers, shared by the kernel-level convolution tests
(test_conv_kernels_gpu.py, test_convlstm_state_gpu.py) and the launch-by-launch network tests
(net_launches_common.py).

The tensor-core arithmetic is fully determined: its operands are `cvt.rn.satfinite` fp16 roundings of fp32 values
(zero / reflection padding, nearest upsampling and the stride-2 phase split are index maps), accumulated in fp32.  The
reference builds the same fp16 operands (clamp to +-65504, then round to nearest), convolves them in float64 and bounds
the difference per element:

    |y - y_ref| <= c * u * sqrt(R) * A * |out_scale| + 4u * (|out_scale * act(z_ref)| + |y_ref|)

with u = 2^-24, R = Cin * KH * KW and A = conv64(|x16|, |w16|) + |b|.  The activations are 1-Lipschitz or better, so the
bound on the pre-activation carries through.  The fp32 path uses the same form with unrounded operands.  Bilinear x2
upsampling is interpolated in fp32 by the kernels: the reference interpolates in float64 without rounding and adds one
fp16 rounding of that operand (tensor cores only), 2^-11 * (1 + 2^-10) * conv64(|x_interp|, |w16|), and the fp32 index
arithmetic of the interpolation, conv64((4 (H + W) + 8) u * max|x| of the channel, |w|).  C_TC = C_FP32 = 4 (see
test_conv_kernels_gpu.py for how they were set).

Every function here works on CPU and CUDA tensors alike."""
import math

import torch
import torch.nn.functional as F

U = 2.0 ** -24
C_TC = 4.0
C_FP32 = 4.0
ACTS = {"none": lambda t: t, "relu": torch.relu, "leaky": lambda t: F.leaky_relu(t, 0.2), "sigmoid": torch.sigmoid,
        "tanh": torch.tanh}


def f16(t):
    """cvt.rn.satfinite.f16.f32 of fp32 values, as float64."""
    return t.float().clamp(-65504.0, 65504.0).half().double()


def _cdiv(a, b):
    return -(-a // b)


def input_domain(x, c, bilinear):
    """x[:, slice] upsampled and padded, float64 (the convolution proper is then a 'valid' one with the stride)."""
    lo = 0 if c["in_slice"] is None else c["in_slice"][0]
    t = x[:, lo:lo + c["cin"]].double()
    if c["upsample"] == 2:
        t = (F.interpolate(t, scale_factor=2, mode="bilinear", align_corners=True) if bilinear
             else t.repeat_interleave(2, 2).repeat_interleave(2, 3))
    ph, pw = c["pad"]
    return F.pad(t, (pw, pw, ph, ph), mode="reflect" if c["pad_mode"] == "reflect" else "constant")


def reference(c, x, w, b, residual, tc):
    """(y_ref, slack, unit) of the convolution `c` (a test_conv_kernels_gpu.spec dict): float64 output, the part of the
    elementwise bound that does not scale with the constant, and u * sqrt(R) * A * |s|, the quantity the constant
    multiplies.  The bound is C * unit + slack."""
    bilinear = c["upsample"] == 2 and c["up_mode"] == "bilinear"
    xi = input_domain(x, c, bilinear)
    wr = f16(w) if tc else w.double()
    if tc and not bilinear:
        xi = f16(xi)
    br = b.double() if b is not None else None
    s = c["stride"]
    z = F.conv2d(xi, wr, br, stride=s)
    mag = F.conv2d(xi.abs(), wr.abs(), br.abs() if br is not None else None, stride=s)
    extra = torch.zeros_like(z)
    if bilinear:
        if tc:
            extra += 2.0 ** -11 * (1 + 2.0 ** -10) * F.conv2d(xi.abs(), wr.abs(), stride=s)
        lo = 0 if c["in_slice"] is None else c["in_slice"][0]
        m = x[:, lo:lo + c["cin"]].double().abs().amax(dim=(2, 3), keepdim=True).expand(-1, -1, c["h"], c["w"])
        d = (4 * (c["h"] + c["w"]) + 8) * U * input_domain(m.contiguous(), dict(c, in_slice=None), False)
        extra += F.conv2d(d, w.double().abs(), stride=s)
    act = ACTS[c["act"]](z) * c["out_scale"]
    y = act.clone()
    if residual is not None:
        y += residual[:, c["res_slice"][0]:c["res_slice"][0] + c["cout"]].double()
    kh, kw = c["k"]
    unit = U * math.sqrt(c["cin"] * kh * kw) * mag * abs(c["out_scale"])
    slack = 4 * U * (act.abs() + y.abs()) + extra * abs(c["out_scale"])
    return y, slack, unit


def bound_ratio(y, y_ref, slack, unit, const):
    """(largest (err - slack) / unit, elements beyond const * unit + slack, max err) of an output y (any float dtype)
    against reference(...)."""
    err = (y.double() - y_ref).abs()
    over = err - slack
    ratio = float((over / unit.clamp_min(1e-300)).max()) if bool((over > 0).any()) else 0.0
    bad = int((err > const * unit + slack).sum())
    return ratio, bad, float(err.max())


def chain_view(ch, n, cin, h, w, pad):
    """Chain.buf as fp16 [n][h + 2 pad_h][w + 2 pad_w][Cp], Cp = Cin rounded up to 64."""
    ph, pw = pad
    hp, wp, cp = h + 2 * ph, w + 2 * pw, _cdiv(cin, 64) * 64
    return ch.buf[:n * hp * wp * cp * 2].view(torch.float16).view(n, hp, wp, cp)


def convlstm_reference(xin, wt, b, prev_cell, const=C_TC):
    """float64 (hidden, cell) of the fused ConvLSTM gate layer on its fp16 operands (xin = the gates' whole input,
    [x | prev_hidden] with a state; wt the matching weight), and their elementwise bounds (test_convlstm_state_gpu.py):
        E_z = c * u * sqrt(R) * A + 4u |z|,  E_sig = E_z / 4 + 8u |sig|,  E_tanh = E_z + 8u |tanh|,
        E_cell = |c_prev| E_rem + |g| E_in + |in| E_g + E_in E_g + 4u (|rem c_prev| + |in g|),
        E_hidden = |tanh(cell)| E_out + |out| (E_cell + 8u |tanh(cell)|) + E_out E_cell + 4u |hidden|."""
    x16, w16 = f16(xin), f16(wt)
    kh, kw = wt.shape[2:]
    z = F.conv2d(x16, w16, b.double(), padding=(kh // 2, kw // 2))
    a = F.conv2d(x16.abs(), w16.abs(), b.double().abs(), padding=(kh // 2, kw // 2))
    ez = const * U * math.sqrt(xin.shape[1] * kh * kw) * a + 4 * U * z.abs()
    return cell_reference(z, ez, prev_cell)


def cell_reference(z, ez, prev_cell):
    """The ConvLSTM cell in float64 on gates z (chunk(4, 1) order in, remember, out, cell) known to within ez, and the
    bounds of hidden and cell (convlstm_reference; ez = 0 for the fp32 cell kernel on its own gates)."""
    zi, zr, zo, zg = z.chunk(4, 1)
    ei, er, eo, eg = ez.chunk(4, 1)
    si, sr, so, tg = torch.sigmoid(zi), torch.sigmoid(zr), torch.sigmoid(zo), torch.tanh(zg)
    e_in, e_rem, e_out = ei / 4 + 8 * U * si, er / 4 + 8 * U * sr, eo / 4 + 8 * U * so
    e_g = eg + 8 * U * tg.abs()
    cp = torch.zeros_like(si) if prev_cell is None else prev_cell.double()
    cell = sr * cp + si * tg
    e_cell = cp.abs() * e_rem + tg.abs() * e_in + si * e_g + e_in * e_g + 4 * U * ((sr * cp).abs() + (si * tg).abs())
    tc_ = torch.tanh(cell)
    hidden = so * tc_
    e_hidden = tc_.abs() * e_out + so * (e_cell + 8 * U * tc_.abs()) + e_out * e_cell + 4 * U * hidden.abs()
    return hidden, cell, e_hidden, e_cell
