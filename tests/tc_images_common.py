"""Decoders of the fused tensor-core IMLP kernels' operand images (csrc/mlp_tc.cu) and the float64 layer-by-layer
checks built on them, shared by test_tc_layers_gpu.py (stand-alone calls on all rows, the fused atlas step) and
test_seg_tc_layers_gpu.py (the segmentation trip's counted calls).  test_tc_layers_gpu.py's docstring states the
references and the per-element bound (a) to (d) these checks apply.
"""
import ctypes as C
import math
import struct

import pytest
import torch

from b200 import _native as N
from b200 import atlas as A
from b200 import synth

DEV = "cuda"
U = 2.0 ** -24
C_TC = 4.0
SPLIT = 2.0 ** -22
FLOOR = 2.0 ** -24
TM, HID = 128, 256
S_ACT, S_W = 16.0, 256.0
ITEM = 16384
CHUNK = 4 * ITEM
ATOM = TM * 128
TILE = 4 * ATOM
MAXL = 16
OFFSETS = 61          # B200_TC_OFFSET_FLOATS
GMAX = 60             # B200_TC_OFFSET_GMAX


def _need_tc():
    if not N.lib().b200_device_supports_tc():
        pytest.skip("no sm_90 device")



# ---------------------------------------------------------------------------------------------------------------
# Mirrors of the image layouts (csrc/mlp_tc.cu atom_off, tile_off, item_off), as fp16 element indices
# ---------------------------------------------------------------------------------------------------------------
def atom_off(m, k):
    r = m & 7
    return (m >> 3) * 1024 + r * 128 + (((k >> 3) ^ r) << 4) + ((k & 7) << 1)


def tile_off(m, col):
    return (col >> 6) * ATOM + atom_off(m, col & 63)


def item_off(n, k):
    return (n >> 3) * 512 + (n & 7) * 64 + ((((k >> 3) ^ (n >> 1)) & 3) << 4) + ((k & 7) << 1)


_IDX = {}


def _index(kind):
    if kind not in _IDX:
        if kind == "item":
            n, k = torch.arange(HID).view(-1, 1), torch.arange(32).view(1, -1)
            off = item_off(n, k)
        else:
            m, col = torch.arange(TM).view(-1, 1), torch.arange(kind).view(1, -1)
            off = tile_off(m, col) if kind == HID else atom_off(m, col)
        _IDX[kind] = (off // 2).flatten().to(DEV)
    return _IDX[kind]


def split16(v):
    """2-term fp16 split of an fp32 tensor as the kernels form it (cvt.rn.satfinite), as int16 bit patterns."""
    hi = v.clamp(-65504.0, 65504.0).half()
    lo = (v - hi.float()).clamp(-65504.0, 65504.0).half()
    return hi.view(torch.int16), lo.view(torch.int16)


def f64(bits):
    return bits.view(torch.float16).double()


def grad_scale(word):
    """s_g of `grad_scales` from the int32 gmax word."""
    mx = struct.unpack("f", struct.pack("i", int(word)))[0]
    e = 0
    if 0.0 < mx < 3.0e38:
        e = math.frexp(mx)[1]
    e = max(-60, min(60, e))
    return 2.0 ** (13 - e)


def pe_freqs(n):
    return torch.tensor([math.pi * 2.0 ** k for k in range(n)], dtype=torch.float32, device=DEV)


class Net:
    """Shape of one network (b200_mlp_layout) and its fp32 parameters."""

    def __init__(self, dims, flat):
        self.in_dim, self.out, self.L, self.pe, self.skips = dims
        self.desc = A.make_desc(self.in_dim, self.out, HID, self.L, self.pe, self.skips)
        self.w_off, self.b_off, self.total = A.mlp_layout(self.desc)
        self.dims = A.layer_dims(self.desc)
        self.enc = 2 * self.in_dim * self.pe if self.pe else self.in_dim
        self.skip = [l > 0 and l in self.skips for l in range(self.L)]
        self.atlas = self.skip[-1]                   # the atlas: PE skips at 4 and the output layer, input gradient
        self.flat = flat

    def weight(self, l, flat=None):
        k, n = self.dims[l]
        return (self.flat if flat is None else flat)[self.w_off[l]:self.w_off[l] + k * n].view(n, k)

    def bias(self, l):
        return self.flat[self.b_off[l]:self.b_off[l] + self.dims[l][1]]

    def tc_layer(self, l):
        return l <= self.L - 2 and (self.pe > 0 or l >= 1)


class Images:
    """The images of one network in the workspace `ws` (uint8), decoded for the global tiles `tiles`."""

    def __init__(self, ws, off, net, tiles):
        self.ws, self.o, self.net = ws, [int(v) for v in off], net
        self.tiles = torch.as_tensor(tiles, dtype=torch.long, device=DEV)
        self.n_tiles = self.o[11] // TM

    def _img(self, base, width, term_stride):
        tb = TM * width * 2
        out = []
        for t in range(2):
            b = base + t * term_stride
            h = self.ws[b:b + self.n_tiles * tb].view(torch.int16).view(self.n_tiles, tb // 2)
            out.append(h[self.tiles][:, _index(width)].reshape(-1, width))
        return out

    def act(self, s):
        return self._img(self.o[3] + s * self.o[8], HID, self.o[9])

    def dz(self, s):
        return self._img(self.o[4] + s * self.o[8], HID, self.o[9])

    def pe(self):
        return self._img(self.o[5], 64, self.o[10])

    def dzl(self):
        return self._img(self.o[6], 64, self.o[10])

    def flags(self, s):
        rows = self.o[11]
        b = self.o[7] + s * rows * 32
        w = self.ws[b:b + rows * 32].view(torch.int16).view(self.n_tiles, TM, 16)[self.tiles].reshape(-1, 16)
        w = w.int() & 0xFFFF
        col = torch.arange(HID, device=DEV)
        return ((w[:, col >> 4] >> (15 - (col & 15))) & 1).bool()

    def _items(self, base, n_chunks):
        it = self.ws[base:base + n_chunks * CHUNK].view(torch.int16).view(n_chunks, 4, ITEM // 2)
        it = it[:, :, _index("item")].view(n_chunks, 4, HID, 32)
        return [it[:, t:t + 2].permute(2, 0, 1, 3).reshape(HID, n_chunks * 64) for t in (0, 2)]

    def w_fwd(self, l):
        return self._items(self.o[0] + self.o[12 + l], self.o[12 + MAXL + l])

    def w_bwd(self, l):
        return self._items(self.o[1] + self.o[12 + 2 * MAXL + l], 4)

    def cst(self, n):
        return self.ws[self.o[2]:self.o[2] + 4 * n].view(torch.float32)


class Worst:
    def __init__(self):
        self.r = {}

    def add(self, what, got, ref, bound):
        """got, ref, bound: float64 tensors; an error where the bound is zero is infinite."""
        assert torch.isfinite(got).all(), f"{what}: non-finite device value"
        err = (got - ref).abs()
        r = torch.where(err == 0, torch.zeros_like(err), err / bound)
        self.r[what] = max(self.r.get(what, 0.0), float(r.max()) if r.numel() else 0.0)

    def exact(self, what, ok):
        if not bool(ok):
            self.r[what] = math.inf

    def report(self, label):
        where = max(self.r, key=self.r.get)
        dw = max((v, k) for k, v in self.r.items() if k.startswith("dW"))
        print(f"{label}: largest error / bound {self.r[where]:.3g} ({where}); weight gradients {dw[0]:.3g} ({dw[1]})")
        bad = {k: v for k, v in self.r.items() if not v <= 1.0}
        assert not bad, (label, bad)
        return self.r[where]


F16_MAX_BITS = 0x7BFF   # 65504: where cvt.rn.satfinite clamps


def check_unsaturated(worst, what, hi):
    """No hi term of an image sits at +-65504: past it the 2-term split keeps only the lo term's 11 bits."""
    worst.exact(f"no saturated hi term in {what}", not bool(((hi & 0x7FFF) == F16_MAX_BITS).any()))


def _mm3(a_hi, a_lo, b_hi, b_lo):
    """sum_k a_hi b_hi + a_lo b_hi + a_hi b_lo  and the same of absolute values: [R, K] x [N, K] -> [R, N]."""
    v = (a_hi + a_lo) @ b_hi.T + a_hi @ b_lo.T
    a = (a_hi.abs() + a_lo.abs()) @ b_hi.abs().T + a_hi.abs() @ b_lo.abs().T
    return v, a


def _bound(K, chain, A):
    return C_TC * U * (math.sqrt(K) + chain) * A


# ---------------------------------------------------------------------------------------------------------------
# (a) weight images and forward constants
# ---------------------------------------------------------------------------------------------------------------
def check_weight_images(im, net, worst):
    L, enc, pe = net.L, net.enc, net.pe > 0
    for l in range(L):
        want_chunks = ((0 if l == 0 else 4) + (1 if pe and (l == 0 or net.skip[l]) else 0)) if net.tc_layer(l) else 0
        worst.exact(f"n_chunks_fwd[{l}]", im.o[12 + MAXL + l] == want_chunks)
        if not want_chunks:
            continue
        W = net.weight(l)
        blocks = [W[:, kc * 64:(kc + 1) * 64] for kc in range(4)] if l > 0 else []
        if pe and (l == 0 or net.skip[l]):
            k0 = 0 if l == 0 else HID
            blocks.append(torch.nn.functional.pad(W[:, k0:k0 + enc], (0, 64 - enc)))
        hi, lo = split16(torch.cat(blocks, 1) * S_W)
        got_hi, got_lo = im.w_fwd(l)
        worst.exact(f"W items of layer {l}", torch.equal(got_hi, hi) and torch.equal(got_lo, lo))
    for l in range(L - 1):
        if l == 0 and not net.atlas:             # the dgrad reads W^T of layer 0 only to reach the atlas input
            continue
        rows = enc if (pe and l == 0) else HID
        WT = torch.zeros(HID, HID, device=DEV)
        WT[:rows] = net.weight(l)[:, :rows].T     # image row = input index k, column = output index n
        hi, lo = split16(WT * S_W)
        got_hi, got_lo = im.w_bwd(l)
        worst.exact(f"W^T items of layer {l}", torch.equal(got_hi, hi) and torch.equal(got_lo, lo))
    k_last = net.dims[L - 1][0]
    parts = [net.bias(l) * S_ACT for l in range(L - 1)]
    if not pe:
        parts.append(net.weight(0).flatten() * S_ACT)
    parts += [net.weight(L - 1).flatten() * (1.0 / S_ACT), net.bias(L - 1)]
    want = torch.cat(parts)
    worst.exact("forward constants", torch.equal(im.cst(want.numel()), want))
    assert want.numel() == (L - 1) * HID + (0 if pe else 3 * HID) + net.out * k_last + net.out


# ---------------------------------------------------------------------------------------------------------------
# (b) forward, layer by layer
# ---------------------------------------------------------------------------------------------------------------
def cst_layout(net):
    k_last = net.dims[-1][0]
    w0 = (net.L - 1) * HID
    wl = w0 + (0 if net.pe else 3 * HID)
    bl = wl + net.out * k_last
    return w0, wl, bl


def encoding_ref(net, inp):
    """float64 sin / cos of the fp32 products in_r b_k, in the kernels' column order, times S_ACT: [R, 64]."""
    R = inp.shape[0]
    ref = torch.zeros(R, 64, dtype=torch.float64, device=DEV)
    if net.atlas:                                   # column 4k + {sin x0, sin x1, cos x0, cos x1}
        arg = (inp[:, None, :2] * pe_freqs(10)[None, :, None]).double()        # [R, 10, 2]
        ref[:, :40] = torch.cat((torch.sin(arg), torch.cos(arg)), 2).reshape(R, 40)
    else:                                           # column 6k + r: r < 3 sin(x_r b_k), else cos(x_{r-3} b_k)
        P = net.pe
        arg = (inp[:, None, :3] * pe_freqs(P)[None, :, None]).double()         # [R, P, 3]
        ref[:, :6 * P] = torch.cat((torch.sin(arg), torch.cos(arg)), 2).reshape(R, 6 * P)
    return ref * S_ACT


def check_forward(im, net, inp, y_dev, worst, y_rows=None):
    """inp: [R, in] fp32 network input of the decoded rows (after in_scale / in_shift); y_dev: [R, out] output."""
    L = net.L
    w0, wl, bl = cst_layout(net)
    cst = im.cst(bl + net.out).double()
    pe_full = None
    if net.pe:
        p_hi, p_lo = im.pe()
        check_unsaturated(worst, "the encoding", p_hi)
        ref = encoding_ref(net, inp)
        pe_full = f64(p_hi) + f64(p_lo)
        worst.add("encoding", pe_full, ref, 4 * U * ref.abs() + SPLIT * ref.abs() + FLOOR)
    for l in range(L - 1):
        bias = cst[l * HID:(l + 1) * HID]
        if not net.tc_layer(l):                     # the plain mapping's layer 0 on CUDA cores (fma chain)
            x3 = inp[:, :3].double()
            w = cst[w0:w0 + 3 * HID].view(HID, 3)
            z = x3 @ w.T + bias
            bound = _bound(3, 3, x3.abs() @ w.abs().T + bias.abs())
        else:
            a_hi, a_lo, K = [], [], 0
            if l > 0:
                h, lo = im.act(l - 1)
                a_hi.append(f64(h)); a_lo.append(f64(lo)); K += HID
            if net.pe and (l == 0 or net.skip[l]):
                h, lo = im.pe()
                a_hi.append(f64(h)); a_lo.append(f64(lo)); K += 64
            b_hi, b_lo = im.w_fwd(l)
            v, a = _mm3(torch.cat(a_hi, 1), torch.cat(a_lo, 1), f64(b_hi), f64(b_lo))
            z = v / S_W + bias
            bound = _bound(K, 3 * K / 16 + 1, a / S_W + bias.abs())
        flags = im.flags(l)
        h, lo = im.act(l)
        check_unsaturated(worst, f"h{l}", h)
        img = f64(h) + f64(lo)
        sure = z.abs() > bound
        worst.exact(f"flags of layer {l}", torch.equal(flags[sure], z[sure] > 0))
        worst.exact(f"zero flag, zero image of layer {l}", bool((img[~flags] == 0).all()))
        worst.add(f"h{l}", img, torch.relu(z), bound + SPLIT * z.abs() + FLOOR)
    # output layer on CUDA cores: the fp32 activations (the image to 22 bits) against W_{L-1} / S_ACT
    k_last = net.dims[-1][0]
    wlast = cst[wl:bl].view(net.out, k_last)
    h, lo = im.act(L - 2)
    v = f64(h) + f64(lo)
    o = v @ wlast[:, :HID].T + cst[bl:bl + net.out]
    a = v.abs() @ wlast[:, :HID].abs().T + cst[bl:bl + net.out].abs()
    if net.atlas:
        o = o + pe_full[:, :40] @ wlast[:, HID:].T
        a = a + pe_full[:, :40].abs() @ wlast[:, HID:].abs().T
    bound = _bound(k_last, k_last / 4 + 3, a) + SPLIT * a + FLOOR * wlast.abs().sum(1)
    ref = torch.tanh(o)
    n = y_dev.shape[0] if y_rows is None else y_rows
    worst.add("y", y_dev[:n].double(), ref[:n], (bound + 4 * U * ref.abs())[:n])


# ---------------------------------------------------------------------------------------------------------------
# (c) backward, layer by layer
# ---------------------------------------------------------------------------------------------------------------
def check_backward(im, net, y_dev, dy_dev, s_g, worst):
    """y_dev, dy_dev: [R, out] fp32 output and output gradient of the decoded rows (zero in padding rows)."""
    L, out = net.L, net.out
    d_hi, d_lo = im.dzl()
    check_unsaturated(worst, "dZ output", d_hi)
    dzl = f64(d_hi) + f64(d_lo)
    y, dy = y_dev.double(), dy_dev.double()
    ref = s_g * dy * (1 - y * y)
    worst.add("dZ output", dzl[:, :out], ref, s_g * 4 * U * dy.abs() * (1 + y * y) + SPLIT * ref.abs() + FLOOR)
    worst.exact("dZ output padding", bool((d_hi[:, out:] == 0).all() and (d_lo[:, out:] == 0).all()))
    # dZ_{L-2} = mask (dz_out W_{L-1}[:, :256]), fp32 fma over the outputs
    W = net.weight(L - 1)[:, :HID].double()
    g = dzl[:, :out] / s_g
    mask = im.flags(L - 2)
    ref = s_g * (g @ W) * mask
    a = s_g * (g.abs() @ W.abs())
    bound = mask * ((C_TC * U * (math.sqrt(out) + out) + SPLIT) * a + SPLIT * ref.abs() + FLOOR)
    h, lo = im.dz(L - 2)
    check_unsaturated(worst, f"dZ{L - 2}", h)
    worst.add(f"dZ{L - 2}", f64(h) + f64(lo), ref, bound)
    # hidden layers: dZ_{l-1} = mask (dZ_l W_l), on the tensor cores with the W^T items
    for l in range(L - 2, 0, -1):
        if l - 1 == 0 and not net.pe:               # the plain mapping keeps dZ_0 on chip (its row sums only)
            continue
        h, lo = im.dz(l)
        b_hi, b_lo = im.w_bwd(l)
        v, a = _mm3(f64(h), f64(lo), f64(b_hi), f64(b_lo))
        mask = im.flags(l - 1)
        ref = v / S_W * mask
        bound = mask * (_bound(HID, 3 * HID / 16 + 1, a / S_W) + SPLIT * ref.abs() + FLOOR)
        h, lo = im.dz(l - 1)
        check_unsaturated(worst, f"dZ{l - 1}", h)
        worst.add(f"dZ{l - 1}", f64(h) + f64(lo), ref, bound)


def check_input_gradient(im, net, s_g, d_in, worst, base=None):
    """The atlas: dPE = dZ_0 W_0 (64 columns) on the tensor cores, then d(in)_e = sum_k b_k (dsin c - dcos s) with
    the partner terms of the device's encoding image.

    base: None when the kernel overwrites d_in with d(in) (stand-alone calls), or (value, bound), float64 [n, 2]
    tensors, when it adds its gradient into a buffer that held `value` to within an absolute `bound`: the fused step
    adds 0.5 d(in) (its atlas input is uv * 0.5 + 0.5) into the loss head's d_uv, with one fp32 rounding of the sum.
    An infinite bound leaves a row only the finiteness check."""
    h, lo = im.dz(0)
    b_hi, b_lo = im.w_bwd(0)
    v, a = _mm3(f64(h), f64(lo), f64(b_hi[:64]), f64(b_lo[:64]))
    dpe, e_dpe = v / (S_W * s_g), _bound(HID, 3 * HID / 16 + 1, a / (S_W * s_g))
    p_hi, p_lo = im.pe()
    pe = (f64(p_hi) + f64(p_lo)) / S_ACT
    bk = pe_freqs(10).double()
    n = d_in.shape[0]
    for e in range(2):
        ds, dc = dpe[:n, e:40:4], dpe[:n, 2 + e:40:4]
        es, ec = e_dpe[:n, e:40:4], e_dpe[:n, 2 + e:40:4]
        s, c = pe[:n, e:40:4], pe[:n, 2 + e:40:4]
        ref = (bk * (ds * c - dc * s)).sum(1)
        bound = (bk * (es * c.abs() + ec * s.abs())).sum(1) + _bound(20, 10, (bk * ((ds * c).abs() + (dc * s).abs())).sum(1))
        got = d_in[:, e].double()
        if base is None:
            worst.add("d_in", got, ref, bound + 1e-300)
        else:
            worst.add("d_in + head", got, base[0][:, e] + 0.5 * ref,
                      base[1][:, e] + 0.5 * bound + U * got.abs() + 1e-300)


# ---------------------------------------------------------------------------------------------------------------
# (d) weight gradients
# ---------------------------------------------------------------------------------------------------------------
def _step_cost(a_cols, b_cols):
    cols = a_cols + b_cols
    return 512.0 if cols >= 512 else (416.0 if cols >= 320 else 340.0)


def wgrad_gemms(net):
    """The GEMMs of one network's work list, in the order of `protos_for_net`: (name, a_cols, b_cols)."""
    g = [(f"dW{l}", HID, HID) for l in range(1, net.L - 1)] + [(f"dW{net.L - 1}", HID, 64)]
    if net.pe:
        g.append(("dW0", HID, 64))
        g += [(f"dW{l} skip", HID, 64) for l in range(1, net.L - 1) if net.skip[l]]
        if net.skip[net.L - 1]:
            g.append((f"dW{net.L - 1} skip", 64, 64))
    return g


def unit_splits(gemms, units):
    """`apportion_items`: units of the work list per GEMM.  gemms: [(a_cols, b_cols, groups)]."""
    cost = [gr * _step_cost(a, b) for a, b, gr in gemms]
    want = [c / sum(cost) * units for c in cost]
    n = [max(1, int(w)) for w in want]
    frac = [w - int(w) for w in want]
    while sum(n) < units:
        best = max(range(len(n)), key=lambda i: (frac[i], -i))
        n[best] += 1
        frac[best] = -1.0
    while sum(n) > units:
        cand = [i for i in range(len(n)) if n[i] > 1]
        if not cand:
            break
        best = max(cand, key=lambda i: (n[i], -i))
        n[best] -= 1
    return n


def check_weight_gradients(im, net, grads, s_g, live_tiles, n_split, worst):
    """Every dW the weight-gradient kernel writes, per element, from the device's dZ and activation images."""
    L, out, enc = net.L, net.out, net.enc
    for (name, a_cols, b_cols), ns in zip(wgrad_gemms(net), n_split):
        tiles = -(-live_tiles // ns)
        K = tiles * TM
        chain = 3 * K / 16 + 2 * min(ns, live_tiles)
        l = int(name.split()[0][2:])
        skip = name.endswith("skip")
        if l == L - 1 and not skip:                  # transposed: M = the last activation, N = the output dZ
            a_img, b_img = im.act(L - 2), im.dzl()
        elif l == L - 1:
            a_img, b_img = im.dzl(), im.pe()
        else:
            a_img = im.dz(l)
            b_img = im.pe() if (skip or l == 0) else im.act(l - 1)
        a_hi, a_lo = f64(a_img[0]), f64(a_img[1])
        b_hi, b_lo = f64(b_img[0]), f64(b_img[1])
        v = (a_hi + a_lo).T @ b_hi + a_hi.T @ b_lo
        a = (a_hi.abs() + a_lo.abs()).T @ b_hi.abs() + a_hi.abs().T @ b_lo.abs()
        ref, bound = v / (s_g * S_ACT), _bound(K, chain, a / (s_g * S_ACT))
        G = net.weight(l, grads).double()
        if l == L - 1 and not skip:
            got, ref, bound = G[:, :HID], ref[:, :out].T, bound[:, :out].T
        elif l == L - 1:
            got, ref, bound = G[:, HID:], ref[:out, :enc], bound[:out, :enc]
        elif skip or l == 0:
            k0 = HID if skip else 0
            got, ref, bound = G[:, k0:k0 + enc], ref[:, :enc], bound[:, :enc]
        else:
            got = G[:, :HID]
        worst.add(name, got, ref, bound)




@pytest.fixture(scope="module")
def wg_units():
    """Units of the weight-gradient work list (two per cluster of two CTAs that fits on the device), read from the
    kernel's last launch after a small fused step."""
    _need_tc()
    H, W, T, B = 24, 40, 6, 300
    data = synth.throughput_set(H, W, T, seed=3)
    tr = A.AtlasTrainer(A.DeviceVideo.from_reference_layout(data, DEV), {"samples_batch": B}, precision=N.PREC_TC,
                        device=DEV)
    tr.indices.copy_(torch.randint(H * W * T, (B,), generator=torch.Generator().manual_seed(2)))
    tr.loss_grad(True)
    torch.cuda.synchronize()
    cycles, shapes = (C.c_longlong * 1024)(), (C.c_int32 * 3072)()
    ctas = N.lib().b200_debug_wgrad(cycles, shapes, 1024)
    assert ctas > 0 and ctas % 2 == 0
    return ctas            # 2 units per cluster of 2 CTAs


# ---------------------------------------------------------------------------------------------------------------
# counted trips: the tiles a launch visits, host counts, hand-built batches on a small video
# ---------------------------------------------------------------------------------------------------------------
SMALL = dict(T=4, H=32, W=48)
FRAME = 1                      # the resident samples' frame: it has both flow directions, rank 0 of 2 owns it
B_SMALL = 400


def tiles_of(n):
    return -(-n // TM)


def live_tiles(cap, groups, cnt, g_fwd, g_bwd):
    """TileIter::init / global_tile on the host: the global tile indices a counted call visits."""
    ct = cap // TM
    gf = g_fwd if 0 <= g_fwd < groups else -1
    gb = g_bwd if 0 <= g_bwd < groups else -1
    t0 = min(ct, tiles_of(cnt[0]))
    tf = min(ct, tiles_of(cnt[5])) if gf >= 0 else t0
    tb = min(ct, tiles_of(cnt[6])) if gb >= 0 else t0
    return [g * ct + t for g in range(groups) for t in range(tf if g == gf else (tb if g == gb else t0))]


def desc_dims(d):
    """Net's dims of a B200MlpDesc."""
    skips = tuple(l for l in range(d.num_layers) if d.skip_mask >> l & 1)
    return (d.input_dim, d.output_dim, d.num_layers, d.pe_freqs, skips)


def host_counts(inds, data, t0, t1, H, W):
    """counters[0], [5], [6]: resident samples of frames [t0, t1) and those of them with a valid forward / backward
    flow."""
    inds = inds.reshape(-1)
    t = inds // (H * W)
    yx = inds % (H * W)
    here = (t >= t0) & (t < t1)
    wf = data["mask_fwd"][yx // W, yx % W, t, 0] != 0
    wb = data["mask_bwd"][yx // W, yx % W, t, 0] != 0
    return int(here.sum()), int((here & wf).sum()), int((here & wb).sum())


def run_trip(tr, it, replay=None):
    """One trip on a workspace filled with 0xFF (eagerly, or by replaying the CUDA graph `replay`).  `it` is what
    the trainer's loss_grad takes: the iteration (SegTrainer) or the global-term switch (AtlasTrainer)."""
    tr._workspace().fill_(0xFF)
    if replay is None:
        tr.loss_grad(it)
    else:
        replay.replay()
    torch.cuda.synchronize()


def small_data(seed=5):
    """32 x 48 x 4 video whose frame FRAME has the four flow-validity classes in turn: pixel p has a valid forward
    flow iff p & 1, a valid backward flow iff p & 2."""
    T, H, W = SMALL["T"], SMALL["H"], SMALL["W"]
    data = synth.throughput_set(H, W, T, seed=seed)
    p = torch.arange(H * W)
    data["mask_fwd"][:, :, FRAME, 0] = (p & 1).float().view(H, W)
    data["mask_bwd"][:, :, FRAME, 0] = ((p >> 1) & 1).float().view(H, W)
    masks = (torch.rand(H, W, T, generator=torch.Generator().manual_seed(seed)) < 0.4).float()
    return data, masks


def small_batch(n_local, n_f, n_b, seed, resident=True):
    """B_SMALL indices: n_local distinct pixels of frame FRAME of which n_f have a valid forward and n_b a valid
    backward flow (none when not `resident`), the rest in frames 2 and 3 (rank 1's)."""
    T, H, W = SMALL["T"], SMALL["H"], SMALL["W"]
    n11 = max(0, n_f + n_b - n_local)
    per_class = {3: n11, 1: n_f - n11, 2: n_b - n11, 0: n_local - n_f - n_b + n11}
    assert min(per_class.values()) >= 0 and max(per_class.values()) <= H * W // 4, per_class
    pix = [c + 4 * j for c, n in per_class.items() for j in range(n)]
    g = torch.Generator().manual_seed(seed)
    local = torch.tensor(pix, dtype=torch.long) + FRAME * H * W
    rest = 2 * H * W + torch.randint(2 * H * W, (B_SMALL - n_local,), generator=g)
    inds = torch.cat((local, rest))
    return inds[torch.randperm(B_SMALL, generator=g)]


def flow_counts(n_local, regime):
    """(n_f, n_b) of a small batch with n_local resident rows: no forward-flow row ("no_fwd"), every resident row
    forward-valid ("all_fwd"), or forward rows a multiple of 128 beside backward rows that are not."""
    if regime == "no_fwd":
        return 0, max(1, n_local // 3)
    if regime == "all_fwd":
        return n_local, n_local // 2
    n_b = max(x for x in range(n_local, 0, -1) if x % TM)
    return n_local // TM * TM, n_b
