"""Thin torch-tensor wrappers over the convolution / RAFT entry points of libb200deflicker.so
(include/b200_deflicker.h).  CUDA tensors only; every call runs on the current stream."""
import ctypes as C
import weakref

import torch

from . import _native as N

ACT = {"none": 0, "relu": 1, "leaky": 2, "sigmoid": 3, "tanh": 4}

# Convolution arithmetic: "fp32" = CUDA-core FFMA (bit-comparable with an fp32 cuDNN/CPU convolution up to
# summation order), "tc" = wgmma with fp16 operands and fp32 accumulation — the operand precision the
# reference itself uses for these layers (fp16 autocast in RAFT, TF32 cuDNN in stage 2).
_conv_precision = "fp32"
_weight_images = {}        # id(weight tensor) -> (weakref to it, {image key (_image_key): packed fp16 images})


def set_conv_precision(mode):
    """'fp32' or 'tc' (TMA-fed wgmma; stride 1 or 2).  Returns the previous mode."""
    global _conv_precision
    if mode not in ("fp32", "tc"):
        raise N.B200Error(f"unknown convolution precision {mode!r}")
    prev, _conv_precision = _conv_precision, mode
    return prev


def conv_precision():
    return _conv_precision


def _images_for(d, w, lstm=False):
    """Packed weight images, cached per weight TENSOR OBJECT (not per address alone: a freed tensor's address is
    reused) and keyed on everything the image depends on: the storage (`w.data = t`, `module.to(...)`), the in-place
    version, the stride, whether the x taps are folded into the channel vector (decided by the upsampling mode
    for a given weight shape) and the row layout (plain, or gate-interleaved for `convlstm` with lstm=True).
    Pass module parameters themselves (conv.weight) to benefit from the cache.
    Writes through `w.data` (`w.data.copy_(t)`) bump no version and keep the storage, so they are not seen: call
    `clear_weight_images()` after them."""
    key = id(w)
    ent = _weight_images.get(key)
    if ent is None or ent[0]() is not w:
        ent = (weakref.ref(w, lambda _r, k=key: _weight_images.pop(k, None)), {})
        _weight_images[key] = ent
    nbytes = N.lib().b200_conv_tma_weight_image_bytes(C.byref(d))
    if nbytes <= 0:
        raise N.B200Error("conv weight image size: invalid descriptor: " + N.last_error())
    sub = (w.data_ptr(), str(w.device), w._version, d.stride, d.upsample_mode, "lstm" if lstm else "plain")
    img = ent[1].get(sub)
    if img is None:
        ent[1].clear()
        img = torch.empty(nbytes, dtype=torch.uint8, device=w.device)
        build = N.lib().b200_convlstm_tma_weight_images if lstm else N.lib().b200_conv_tma_weight_images
        N.check(build(C.byref(d), N.ptr(w), N.ptr(img), N.current_stream()), "conv weight images")
        ent[1][sub] = img
    assert img.numel() == nbytes, "cached weight image does not match the convolution's layout"
    return img


def clear_weight_images():
    """Drop the cached packed weight images (needed after writes through `w.data`, which the cache cannot see).
    Only when no captured CUDA graph still refers to them."""
    _weight_images.clear()


def _check(t):
    if t is not None and (not t.is_cuda or t.dtype != torch.float32 or not t.is_contiguous()):
        raise N.B200Error("expected a contiguous fp32 CUDA tensor (no CPU fallback)")
    return t


_chain_buffers = {}        # (device, n, cin, h, w, kh, kw, ph, pw, tag) -> zero-initialised packed-input buffer


class Chain:
    """The packed fp16 NHWC input of ONE consumer convolution (stride 1, zero or reflection padding, Cin * KW > 64), filled directly
    by the epilogues of the convolutions that produce it (`conv2d(..., chain_out=chain)`), then consumed by
    `conv2d(chain, w, ...)`: no fp32 tensor in between and no repack kernel.  wgmma path only.  Buffers are cached per
    geometry and zeroed once: producers overwrite the whole interior every time, halo and channel padding stay zero."""

    def __init__(self, n, cin, h, w, kernel, pad, device, tag="", pad_mode="zeros"):
        kh, kw = kernel
        ph, pw = (pad, pad) if isinstance(pad, int) else pad
        self.n, self.cin, self.h, self.w, self.pad_mode = n, cin, h, w, pad_mode
        self.desc = N.ConvDesc(n, cin, h, w, cin, 0, 8, kh, kw, 1, ph, pw, 1 if pad_mode == "reflect" else 0, 1, 8, 0, 0, 1.0,
                               0, 0, 0)
        if not N.lib().b200_conv_tma_chainable(C.byref(self.desc)):
            raise N.B200Error("this convolution cannot consume a chained (pre-packed) input")
        # `tag` separates buffers of equal geometry that are alive at the same time (a consumer whose own output is
        # chained into another buffer of the same shape must not read and write one allocation)
        key = (str(device), n, cin, h, w, kh, kw, ph, pw, pad_mode, tag)
        buf = _chain_buffers.get(key)
        if buf is None:
            nbytes = int(N.lib().b200_conv_tma_workspace_bytes(C.byref(self.desc)))
            buf = _chain_buffers[key] = torch.zeros(nbytes, dtype=torch.uint8, device=device)
        self.buf = buf

    @staticmethod
    def available():
        return _conv_precision == "tc"


def clear_chain_buffers():
    """Drop the cached packed-input buffers (they persist per geometry: ~1.2 GB for the stage-2 networks at 1088x1920).
    Only when no captured CUDA graph still refers to them."""
    _chain_buffers.clear()


def conv2d(x, w, b=None, stride=1, pad=(0, 0), pad_mode="zeros", act="none", upsample=1, out=None, out_c_off=0,
           in_slice=None, residual=None, res_c_off=0, out_scale=1.0, precision=None, upsample_mode="nearest",
           chain_out=None, chain_c_off=0, keep_fp32=True):
    """y = act(conv(pad(upsample(x[:, in_slice]))) + b) * out_scale (+ residual[:, res slice]) written into
    out[:, out_c_off:out_c_off+Cout] (allocated when None).  Restates nn.Conv2d / ReflectionPad2d / Upsample.
    `x` may be a `Chain` (input already packed by its producers); `chain_out` additionally writes the result into the
    consumer's packed input at channel `chain_c_off`, and with keep_fp32=False the fp32 tensor is not produced (returns
    None).  With precision 'tc' (and whenever `x` or `chain_out` is a `Chain`) the convolution runs on the wgmma
    path, which takes stride 1 or 2 only: any other stride raises B200Error rather than changing the arithmetic."""
    _check(w); _check(b); _check(residual)
    mode = _conv_precision if precision is None else precision
    if mode not in ("fp32", "tc"):
        raise N.B200Error(f"unknown convolution precision {mode!r}")
    packed_in = isinstance(x, Chain)
    tc = mode == "tc" or packed_in or chain_out is not None
    if not packed_in:
        _check(x)
    bilinear = 0
    if upsample_mode == "bilinear":
        if upsample != 2:
            raise N.B200Error("bilinear upsampling is x2 only")
        if tc:
            bilinear = 1                                  # fused into the fp16 repack of b200_conv2d_tma_chain
        else:                                             # explicit nn.Upsample kernel, then a plain convolution
            if in_slice is not None:
                x = x[:, in_slice[0]:in_slice[1]].contiguous()
                in_slice = None
            x, upsample = upsample_bilinear2(x), 1
    elif upsample_mode != "nearest":
        raise N.B200Error(f"unknown upsample mode {upsample_mode!r}")
    if packed_in:
        if in_slice is not None or stride != 1 or upsample != 1 or pad_mode != x.pad_mode:
            raise N.B200Error("a chained input feeds a plain stride-1 convolution of the whole tensor, padded as declared")
        n, c_total, h, wd = x.n, x.cin, x.h, x.w
        dev = x.buf.device
    else:
        n, c_total, h, wd = x.shape
        dev = x.device
    c_off, cin = (0, c_total) if in_slice is None else (in_slice[0], in_slice[1] - in_slice[0])
    cout, cin_w, kh, kw = w.shape
    if cin_w != cin:
        raise N.B200Error(f"weight expects {cin_w} input channels, got {cin}")
    ph, pw = (pad, pad) if isinstance(pad, int) else pad
    hu, wu = h * upsample, wd * upsample
    oh, ow = (hu + 2 * ph - kh) // stride + 1, (wu + 2 * pw - kw) // stride + 1
    if keep_fp32 or chain_out is None:
        if out is None:
            out = torch.empty(n, cout, oh, ow, dtype=torch.float32, device=dev)
        _check(out)
    else:
        out = None
    d = N.ConvDesc(n, cin, h, wd, c_total, c_off, cout, kh, kw, stride, ph, pw, 1 if pad_mode == "reflect" else 0, upsample,
                   out.shape[1] if out is not None else cout, out_c_off if out is not None else 0, ACT[act], float(out_scale),
                   residual.shape[1] if residual is not None else 0, res_c_off, bilinear)
    if not tc:
        N.check(N.lib().b200_conv2d(C.byref(d), N.ptr(x), N.ptr(w), N.ptr(b), N.ptr(residual), N.ptr(out),
                                    N.current_stream()), "b200_conv2d")
        return out
    if packed_in and (x.desc.KH, x.desc.KW, x.desc.pad_h, x.desc.pad_w) != (kh, kw, ph, pw):
        raise N.B200Error("the chained input was packed for another filter geometry")
    ws, nbytes = None, 0
    if not packed_in:
        nbytes = N.lib().b200_conv_tma_workspace_bytes(C.byref(d))
        if nbytes <= 0:
            raise N.B200Error("b200_conv_tma_workspace_bytes: " + N.last_error())
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    N.check(N.lib().b200_conv2d_tma_chain(
        C.byref(d), None if packed_in else N.ptr(x), N.ptr(x.buf) if packed_in else None, N.ptr(_images_for(d, w)),
        N.ptr(b), N.ptr(residual), N.ptr(out), N.ptr(chain_out.buf) if chain_out is not None else None,
        C.byref(chain_out.desc) if chain_out is not None else None, int(chain_c_off), N.ptr(ws), nbytes,
        N.current_stream()), "b200_conv2d_tma_chain")
    return out


def maxpool2(x):
    _check(x)
    n, c, h, w = x.shape
    y = torch.empty(n, c, h // 2, w // 2, dtype=torch.float32, device=x.device)
    N.check(N.lib().b200_maxpool2(N.ptr(x), N.ptr(y), n * c, h, w, N.current_stream()), "b200_maxpool2")
    return y


def upsample_bilinear2(x, out=None, out_c_off=0):
    _check(x)
    n, c, h, w = x.shape
    if out is None:
        out = torch.empty(n, c, 2 * h, 2 * w, dtype=torch.float32, device=x.device)
    N.check(N.lib().b200_upsample_bilinear2(N.ptr(x), N.ptr(out), n, c, h, w, out.shape[1], out_c_off,
                                            N.current_stream()), "b200_upsample_bilinear2")
    return out


def gru_gate(a, b, c=None, out=None, mode=0):
    """mode 0: out[:, :C] = a*b ; mode 1: (1-a)*b + a*c."""
    _check(a); _check(b); _check(c)
    n = a.shape[0]
    per = a.numel() // n
    if out is None:
        out = torch.empty_like(a)
    N.check(N.lib().b200_gru_gate(N.ptr(a), N.ptr(b), N.ptr(c), N.ptr(out), per, n, out.numel() // n, mode,
                                  N.current_stream()), "b200_gru_gate")
    return out


def convlstm_zero_state(gates, want_cell=True):
    _check(gates)
    n, c4, h, w = gates.shape
    hidden = torch.empty(n, c4 // 4, h, w, dtype=torch.float32, device=gates.device)
    cell = torch.empty_like(hidden) if want_cell else None
    N.check(N.lib().b200_convlstm_zero_state(N.ptr(gates), N.ptr(hidden), N.ptr(cell), n, c4 // 4, h, w,
                                             N.current_stream()), "b200_convlstm_zero_state")
    return hidden, cell


def _check_state(prev_state, shape, device):
    """A ConvLSTM state: (hidden, cell), both contiguous fp32 CUDA tensors of `shape` on `device`."""
    if not isinstance(prev_state, (tuple, list)) or len(prev_state) != 2:
        raise N.B200Error("prev_state must be a (hidden, cell) pair")
    for name, t in zip(("hidden", "cell"), prev_state):
        if not isinstance(t, torch.Tensor):
            raise N.B200Error(f"prev_state {name} is not a tensor")
        _check(t)
        if tuple(t.shape) != tuple(shape):
            raise N.B200Error(f"prev_state {name} has shape {tuple(t.shape)}, expected {tuple(shape)}")
        if t.device != torch.device(device):
            raise N.B200Error(f"prev_state {name} is on {t.device}, the input on {device}")
    return prev_state


def convlstm_cell(gates, prev_cell=None, want_cell=True):
    """ConvLSTM cell on fp32 gates (N, 4C, H, W), pre-activation in chunk(4, 1) order -> (hidden, cell); prev_cell
    None is the zero state (what convlstm_zero_state computes)."""
    _check(gates)
    n, c4, h, w = gates.shape
    if prev_cell is not None:
        _check(prev_cell)
        if tuple(prev_cell.shape) != (n, c4 // 4, h, w) or prev_cell.device != gates.device:
            raise N.B200Error("prev_cell does not match the gates")
    hidden = torch.empty(n, c4 // 4, h, w, dtype=torch.float32, device=gates.device)
    cell = torch.empty_like(hidden) if want_cell else None
    N.check(N.lib().b200_convlstm_cell(N.ptr(gates), N.ptr(prev_cell), N.ptr(hidden), N.ptr(cell), n, c4 // 4, h, w,
                                       N.current_stream()), "b200_convlstm_cell")
    return hidden, cell


def convlstm(x, weight, bias, prev_state=None, want_cell=True):
    """ConvLSTM step on the tensor cores (nn.Conv2d gates with 'same' zero padding, then the cell update fused into
    the gate convolution's epilogue; the 4C gate channels are never stored) -> fresh (hidden, cell) tensors, cell None
    with want_cell=False.  `weight` (4C, Cin, KH, KW) and `bias` (4C) are the reference's Gates parameters unchanged.
    prev_state None: the zero state, `weight` holds only the input half (Cin = channels of x).  With a state
    (hidden, cell), each (N, C, H, W): `weight` is the full (4C, 2C, KH, KW) tensor and `x` is either a tensor of C
    channels or a `Chain` of 2C channels whose first C its producers wrote; the previous hidden state fills the rest."""
    _check(weight); _check(bias)
    c4, cin, kh, kw = weight.shape
    if c4 % 32:
        raise N.B200Error(f"ConvLSTM gates: {c4} output channels are not 4 * C with C a multiple of 8")
    c = c4 // 4
    packed_in = isinstance(x, Chain)
    if packed_in:
        n, cx, h, wd, dev = x.n, x.cin, x.h, x.w, x.buf.device
        if x.pad_mode != "zeros" or (x.desc.KH, x.desc.KW, x.desc.pad_h, x.desc.pad_w) != (kh, kw, kh // 2, kw // 2):
            raise N.B200Error("the chained input was packed for another filter geometry")
    else:
        _check(x)
        n, cx, h, wd = x.shape
        dev = x.device
    if prev_state is not None:
        _check_state(prev_state, (n, c, h, wd), dev)
        if cin != 2 * c or cx != (2 * c if packed_in else c):
            raise N.B200Error(f"ConvLSTM with a state: weight of {cin} input channels, input of {cx}, hidden of {c}")
        if packed_in:
            N.check(N.lib().b200_conv_tma_pack_chain(C.byref(x.desc), N.ptr(prev_state[0]), c, N.ptr(x.buf), c,
                                                     N.current_stream()), "b200_conv_tma_pack_chain")
        else:
            x, cx = torch.cat((x, prev_state[0]), 1), 2 * c
    elif cin != cx:
        raise N.B200Error(f"weight expects {cin} input channels, got {cx}")
    d = N.ConvDesc(n, cx, h, wd, cx, 0, c4, kh, kw, 1, kh // 2, kw // 2, 0, 1, c4, 0, 0, 1.0, 0, 0, 0)
    ws, nbytes = None, 0
    if not packed_in:
        nbytes = N.lib().b200_conv_tma_workspace_bytes(C.byref(d))
        if nbytes <= 0:
            raise N.B200Error("b200_conv_tma_workspace_bytes: " + N.last_error())
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    hidden = torch.empty(n, c, h, wd, dtype=torch.float32, device=dev)
    cell = torch.empty_like(hidden) if want_cell else None
    N.check(N.lib().b200_convlstm_tma(
        C.byref(d), None if packed_in else N.ptr(x), N.ptr(x.buf) if packed_in else None,
        N.ptr(_images_for(d, weight, lstm=True)), N.ptr(bias), N.ptr(prev_state[1]) if prev_state is not None else None,
        N.ptr(hidden), N.ptr(cell), N.ptr(ws), nbytes, N.current_stream()), "b200_convlstm_tma")
    return hidden, cell


def convex_upsample(flow, mask):
    _check(flow); _check(mask)
    n, _, h, w = flow.shape
    out = torch.empty(n, 2, 8 * h, 8 * w, dtype=torch.float32, device=flow.device)
    N.check(N.lib().b200_convex_upsample(N.ptr(flow), N.ptr(mask), N.ptr(out), n, h, w, N.current_stream()),
            "b200_convex_upsample")
    return out


def corr_build(fmap1, fmap2, impl="tc", out=None):
    """fmaps (1, C, H8, W8) -> flat pyramid tensor (level 0 [HW][H8][W8] then 3 pooled levels).
    impl 'tc': wgmma with (hi, lo) fp16 operand pairs (fp32-grade, like the reference's fp32 matmul);
    'simt': fp32 CUDA-core GEMM."""
    _check(fmap1); _check(fmap2)
    if fmap1.shape[0] != 1:
        raise N.B200Error("correlation kernels take batch 1 (the reference runs one frame pair at a time)")
    return corr_build_batch(fmap1, fmap2, impl, out).view(-1)


def corr_build_batch(fmap1, fmap2, impl="tc", out=None):
    """fmaps (B, C, H8, W8) -> (B, b200_corr_pyramid_floats) pyramids, each the bits corr_build returns for its pair."""
    _check(fmap1); _check(fmap2)
    b, c, h, w = fmap1.shape
    if fmap2.shape != fmap1.shape:
        raise N.B200Error("corr_build: fmap1 and fmap2 differ in shape")
    n_pyr = int(N.lib().b200_corr_pyramid_floats(h, w))
    pyr = out if out is not None else torch.empty(b, n_pyr, dtype=torch.float32, device=fmap1.device)
    _check(pyr)
    if pyr.numel() != b * n_pyr:
        raise N.B200Error("corr_build: `out` has the wrong size")
    if impl == "tc":
        nbytes = N.lib().b200_corr_build_tc_batch_workspace_bytes(b, c, h, w)
        if nbytes <= 0:
            raise N.B200Error("b200_corr_build_tc_batch_workspace_bytes: bad arguments")
        ws = torch.empty(nbytes, dtype=torch.uint8, device=fmap1.device)
        N.check(N.lib().b200_corr_build_tc_batch(N.ptr(fmap1), N.ptr(fmap2), b, c, h, w, N.ptr(pyr), N.ptr(ws), nbytes,
                                                 N.current_stream()), "b200_corr_build_tc_batch")
    elif impl == "simt":
        N.check(N.lib().b200_corr_build_batch(N.ptr(fmap1), N.ptr(fmap2), b, c, h, w, N.ptr(pyr), N.current_stream()),
                "b200_corr_build_batch")
    else:
        raise N.B200Error(f"unknown correlation builder {impl!r}")
    return pyr.view(b, n_pyr)


def corr_lookup(pyr, coords, radius=4):
    _check(pyr); _check(coords)
    b, _, h, w = coords.shape
    out = torch.empty(b, 4 * (2 * radius + 1) ** 2, h, w, dtype=torch.float32, device=coords.device)
    N.check(N.lib().b200_corr_lookup(N.ptr(pyr), N.ptr(coords), N.ptr(out), b, h, w, radius, N.current_stream()),
            "b200_corr_lookup")
    return out


def corr_lookup_batch(pyr, coords, radius=4):
    """coords (B, 2, H8, W8) on the (B, pyramid floats) pyramids of corr_build_batch -> (B, 4 (2r+1)^2, H8, W8), one
    launch for the batch."""
    _check(pyr); _check(coords)
    b, _, h, w = coords.shape
    if pyr.numel() != b * int(N.lib().b200_corr_pyramid_floats(h, w)):
        raise N.B200Error("corr_lookup_batch: the pyramids were built for another batch or geometry")
    out = torch.empty(b, 4 * (2 * radius + 1) ** 2, h, w, dtype=torch.float32, device=coords.device)
    N.check(N.lib().b200_corr_lookup_batch(N.ptr(pyr), N.ptr(coords), N.ptr(out), b, h, w, radius, N.current_stream()),
            "b200_corr_lookup_batch")
    return out


def corr_alt_build(fmap1, fmap2, out=None):
    """fmaps (1, C, H8, W8) -> the state of the on-the-fly correlation (b200_corr_alt_floats floats: fmap1 and the
    four average-pooled levels of fmap2, pixel-major).  No all-pairs volume: O(C * H8 * W8) memory."""
    _check(fmap1); _check(fmap2)
    if fmap1.shape[0] != 1 or fmap2.shape != fmap1.shape:
        raise N.B200Error("correlation kernels take batch 1 (the reference runs one frame pair at a time)")
    return corr_alt_build_batch(fmap1, fmap2, out).view(-1)


def corr_alt_build_batch(fmap1, fmap2, out=None):
    """fmaps (B, C, H8, W8) -> (B, b200_corr_alt_floats) states, each the bits corr_alt_build returns for its pair."""
    _check(fmap1); _check(fmap2)
    b, c, h, w = fmap1.shape
    if fmap2.shape != fmap1.shape:
        raise N.B200Error("corr_alt_build: fmap1 and fmap2 differ in shape")
    n = int(N.lib().b200_corr_alt_floats(c, h, w))
    if n <= 0:
        raise N.B200Error(f"corr_alt_build: feature maps of {c} channels at {h}x{w} are not supported")
    state = out if out is not None else torch.empty(b, n, dtype=torch.float32, device=fmap1.device)
    _check(state)
    if state.numel() != b * n:
        raise N.B200Error("corr_alt_build: `out` has the wrong size")
    N.check(N.lib().b200_corr_alt_build_batch(N.ptr(fmap1), N.ptr(fmap2), b, c, h, w, N.ptr(state), N.current_stream()),
            "b200_corr_alt_build_batch")
    return state.view(b, n)


def corr_alt_lookup(state, coords, dim, radius=4):
    """What corr_lookup returns on the pyramid of the same feature maps (dim channels), computed from the state of
    corr_alt_build: coords (1, 2, H8, W8) -> (1, 4 (2r+1)^2, H8, W8)."""
    _check(state); _check(coords)
    b, _, h, w = coords.shape
    if state.numel() != int(N.lib().b200_corr_alt_floats(dim, h, w)):
        raise N.B200Error("corr_alt_lookup: the state was built for another geometry")
    out = torch.empty(b, 4 * (2 * radius + 1) ** 2, h, w, dtype=torch.float32, device=coords.device)
    N.check(N.lib().b200_corr_alt_lookup(N.ptr(state), N.ptr(coords), N.ptr(out), dim, b, h, w, radius,
                                         N.current_stream()), "b200_corr_alt_lookup")
    return out


def corr_alt_lookup_batch(state, coords, dim, radius=4):
    """corr_alt_lookup for B pairs at once: coords (B, 2, H8, W8) on the (B, floats) states of corr_alt_build_batch."""
    _check(state); _check(coords)
    b, _, h, w = coords.shape
    if state.numel() != b * int(N.lib().b200_corr_alt_floats(dim, h, w)):
        raise N.B200Error("corr_alt_lookup_batch: the states were built for another batch or geometry")
    out = torch.empty(b, 4 * (2 * radius + 1) ** 2, h, w, dtype=torch.float32, device=coords.device)
    N.check(N.lib().b200_corr_alt_lookup_batch(N.ptr(state), N.ptr(coords), N.ptr(out), dim, b, h, w, radius,
                                               N.current_stream()), "b200_corr_alt_lookup_batch")
    return out


def instance_norm(x, eps=1e-5, relu=False):
    _check(x)
    n, c, h, w = x.shape
    y = torch.empty_like(x)
    N.check(N.lib().b200_instance_norm(N.ptr(x), N.ptr(y), n * c, h * w, eps, 1 if relu else 0, N.current_stream()),
            "b200_instance_norm")
    return y


def add_relu(a, b):
    _check(a); _check(b)
    out = torch.empty_like(a)
    N.check(N.lib().b200_add_relu(N.ptr(a), N.ptr(b), N.ptr(out), a.numel(), N.current_stream()), "b200_add_relu")
    return out
