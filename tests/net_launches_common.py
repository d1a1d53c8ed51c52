"""Launch-by-launch checks of the convolutional networks (stage 2's UNet and TransformNet, RAFT's BasicEncoder and
BasicUpdateBlock, convex upsampling), shared by test_net_launches_cpu.py and test_net_launches_gpu.py.

The networks are restated here as dataflows, one function each, written from the reference's module structure
(oracle/stage2_oracle.py, convlstm_state_common.py, oracle/flow_oracle.py and the reference's BasicEncoder), not from
the implementation's wiring.  A dataflow calls one `dev` method per reference layer (a convolution with its activation,
scale, residual add and batch norm; a ConvLSTM step; a pooling, instance norm, GRU gate or convex upsampling) and
assembles each layer's input from the outputs of the layers that feed it in the reference (`cat`, slices, and the fp32
glue both sides compute with torch: the cnet split into tanh / relu, coords1 - coords0, coords1 + delta).

Two devices run the same dataflows:

- `ExactDevice` evaluates every layer in float64 on the CPU; the CPU test checks that the dataflows then reproduce the
  oracles and the reference's RAFT fixture.
- `LaunchChecker` matches every layer with the launch a `Recorder` captured while the real module ran (by parameter
  identity, merged and folded weights resolved to their source parameters), and returns that launch's recorded device
  output, so that each layer is checked on the device's own operands:
  a. the launch's operand equals the assembled input bit for bit: exactly where the kernel reads fp32, as
     rn_f16(satfinite(.)) where it reads a chained packed input, whose halo must be zero or mirrored (as the padding
     mode says) and whose channel padding must be zero; residuals, recurrent states and GRU gate operands exactly;
  b. the launch's output against float64 on those operands: convolutions within the conv_common bound (one more fp16
     rounding for an output stored only to a chain), the ConvLSTM within the bound of test_convlstm_state_gpu.py,
     maxpool2 / add_relu / gru_gate mode 0 exactly, gru_gate mode 1 within 4u (|h| + |q|), instance norm within the
     bound of test_instance_norm and convex upsampling within that of test_convex_upsample;
  c. host-built weights: a merged weight equals the torch.cat of its sources, the input half of the ConvLSTM gates its
     slice, exactly; a weight or bias folded with batch norm lies within 5u |w64| (weight) and
     6u |(b - mean) s| + 2u |b64| (bias) of the float64 fold, s = gamma / sqrt(var + eps);
  d. every launch is matched exactly once (a merged launch by row ranges that tile its output channels), and each
     launch comes after the launches whose outputs feed it."""
import inspect

import torch
import torch.nn.functional as F
from torch.utils.weak import WeakIdKeyDictionary

from conv_common import C_FP32, C_TC, U, bound_ratio, cell_reference, chain_view, convlstm_reference, reference
from oracle import flow_oracle as FO

FNS = ("conv2d", "convlstm", "convlstm_zero_state", "convlstm_cell", "maxpool2", "gru_gate", "instance_norm",
       "add_relu", "upsample_bilinear2", "convex_upsample")


# ---------------------------------------------------------------------------------------------------------------
# Dataflows (reference structure)
# ---------------------------------------------------------------------------------------------------------------
def unet(dev, p, x):
    """UNet.forward (network_filter.py:54-75)."""
    def block(name, pre, t):
        t = dev.conv(f"{p}{name}.{pre}conv1", t, pad=1, act="relu")
        return dev.conv(f"{p}{name}.{pre}conv2", t, pad=1, act="relu")

    def up(i, t):
        return dev.conv(f"{p}upconv{i}.1", t, pad=1, up="bilinear")

    e1 = block("encoder1", "enc1", x)
    e2 = block("encoder2", "enc2", dev.maxpool(e1))
    e3 = block("encoder3", "enc3", dev.maxpool(e2))
    e4 = block("encoder4", "enc4", dev.maxpool(e3))
    bt = block("bottleneck", "bottleneck", dev.maxpool(e4))
    d4 = block("decoder4", "dec4", dev.cat([up(4, bt), e4]))
    d3 = block("decoder3", "dec3", dev.cat([up(3, d4), e3]))
    d2 = block("decoder2", "dec2", dev.cat([up(2, d3), e2]))
    d1 = block("decoder1", "dec1", dev.cat([up(1, d2), e1]))
    return dev.conv(p + "conv", d1)


def transformnet(dev, p, X, state, blocks=5):
    """TransformNet.forward (network_local.py:88-115) with ConvLSTM.forward (:18-53); state None is the zero state
    (hidden and cell zero).  Returns (Y, (hidden, cell))."""
    def rc(name, t, k, stride=1, up=None, act="leaky", residual=None):
        return dev.conv(p + name + ".conv2d", t, stride=stride, pad=k // 2, pad_mode="reflect", act=act, up=up,
                        residual=residual)

    e1a = rc("conv1a", dev.glue(lambda t: t[:, :6], X), 7)
    e1b = rc("conv1b", dev.glue(lambda t: t[:, 6:], X), 7)
    e2a = rc("conv2a", e1a, 3, 2)
    e2b = rc("conv2b", e1b, 3, 2)
    rb = rc("conv3", dev.cat([e2a, e2b]), 3, 2)
    for b in range(blocks):
        t = rc(f"ResBlocks.{b}.conv1", rb, 3)
        rb = rc(f"ResBlocks.{b}.conv2", t, 3, act="none", residual=rb)
    h0, c0 = state if state is not None else (dev.glue(torch.zeros_like, rb), None)
    hidden, cell = dev.lstm(p + "convlstm.Gates", dev.cat([rb, h0]), c0)
    d2 = rc("deconv1", hidden, 3, up="nearest")
    d1 = rc("deconv2", dev.cat([d2, e2a]), 3, up="nearest")
    y = rc("deconv3", dev.cat([d1, e1a]), 7, act="tanh")
    return y, (hidden, cell)


def encoder(dev, p, x, norm):
    """BasicEncoder.forward (core/extractor.py:118-192) with ResidualBlock (:6-57), norm 'instance' or 'batch'
    (eval mode)."""
    def cn(conv, nrm, t, stride, pad, relu=True):
        if norm == "batch":
            return dev.conv(p + conv, t, stride=stride, pad=pad, act="relu" if relu else "none", bn=p + nrm)
        return dev.inorm(dev.conv(p + conv, t, stride=stride, pad=pad), relu)

    x = cn("conv1", "norm1", x, 2, 3)
    for li, stride in ((1, 1), (2, 2), (3, 2)):
        for bi in (0, 1):
            q = f"layer{li}.{bi}."
            s = stride if bi == 0 else 1
            y = cn(q + "conv1", q + "norm1", x, s, 1)
            y = cn(q + "conv2", q + "norm2", y, 1, 1)
            if s != 1:
                x = cn(q + "downsample.0", q + "norm3", x, s, 0, relu=False)
            x = dev.add_relu(x, y)
    return dev.conv(p + "conv2", x)


def update_block(dev, p, net, inp, corr, flow):
    """BasicUpdateBlock.forward (core/update.py:127-136): BasicMotionEncoder, SepConvGRU, FlowHead, mask head."""
    cor = dev.conv(p + "encoder.convc1", corr, act="relu")
    cor = dev.conv(p + "encoder.convc2", cor, pad=1, act="relu")
    flo = dev.conv(p + "encoder.convf1", flow, pad=3, act="relu")
    flo = dev.conv(p + "encoder.convf2", flo, pad=1, act="relu")
    out = dev.conv(p + "encoder.conv", dev.cat([cor, flo]), pad=1, act="relu")
    x = dev.cat([inp, dev.cat([out, flow])])
    h = net
    for tag, pad in (("1", (0, 2)), ("2", (2, 0))):
        hx = dev.cat([h, x])
        z = dev.conv(p + "gru.convz" + tag, hx, pad=pad, act="sigmoid")
        r = dev.conv(p + "gru.convr" + tag, hx, pad=pad, act="sigmoid")
        q = dev.conv(p + "gru.convq" + tag, dev.cat([dev.gru_rh(r, h), x]), pad=pad, act="tanh")
        h = dev.gru_mix(z, h, q)
    delta = dev.conv(p + "flow_head.conv2", dev.conv(p + "flow_head.conv1", h, pad=1, act="relu"), pad=1)
    mask = dev.conv(p + "mask.2", dev.conv(p + "mask.0", h, pad=1, act="relu"), scale=0.25)
    return h, mask, delta


def refine(dev, p, cnet, corr_at, coords0, iters):
    """RAFT's refinement (core/raft.py:109-148, test mode) from the context encoder's output: `corr_at(it, coords1)` is
    the correlation lookup of iteration `it`.  Returns (flow_low, flow_up)."""
    net = dev.glue(lambda t: torch.tanh(t[:, :128]), cnet)
    inp = dev.glue(lambda t: torch.relu(t[:, 128:]), cnet)
    coords1 = coords0
    mask = None
    for it in range(iters):
        corr = corr_at(it, coords1)
        flow = dev.glue(torch.sub, coords1, coords0)
        net, mask, delta = update_block(dev, p, net, inp, corr, flow)
        coords1 = dev.glue(torch.add, coords1, delta)
    flow_low = dev.glue(torch.sub, coords1, coords0)
    return flow_low, dev.convex(flow_low, mask)


# ---------------------------------------------------------------------------------------------------------------
# Dependency bookkeeping shared by both devices
# ---------------------------------------------------------------------------------------------------------------
class _Deps:
    """Tracks, for every tensor a dataflow holds, the latest launch its value depends on (-1: an input)."""

    def __init__(self):
        self._dep = WeakIdKeyDictionary()

    def dep(self, *ts):
        return max([self._dep.get(t, -1) for t in ts if isinstance(t, torch.Tensor)] + [-1])

    def mark(self, t, idx):
        self._dep[t] = idx
        return t

    def cat(self, ts):
        return self.mark(torch.cat(ts, 1), self.dep(*ts))

    def glue(self, fn, *ts):
        return self.mark(fn(*ts), self.dep(*ts))


def _bn_fold64(norm, conv_w, conv_b):
    """float64 fold of conv -> eval-mode BatchNorm2d: (weight, bias, s)."""
    s = norm["weight"].double() / torch.sqrt(norm["running_var"].double() + 1e-5)
    return conv_w.double() * s.view(-1, 1, 1, 1), (conv_b.double() - norm["running_mean"].double()) * s + \
        norm["bias"].double(), s


# ---------------------------------------------------------------------------------------------------------------
# Float64 device (CPU test)
# ---------------------------------------------------------------------------------------------------------------
class ExactDevice(_Deps):
    """Every layer in float64, as the reference defines it.  `sd`: the modules' state_dict with the dataflow prefixes."""

    def __init__(self, sd):
        super().__init__()
        self.sd = {k: v.double() for k, v in sd.items()}

    def conv(self, name, x, stride=1, pad=0, pad_mode="zeros", act="none", up=None, scale=1.0, residual=None, bn=None):
        w, b = self.sd[name + ".weight"], self.sd.get(name + ".bias")
        x = x.double()
        if up == "bilinear":
            x = F.interpolate(x, scale_factor=2, mode="bilinear", align_corners=True)
        elif up == "nearest":
            x = F.interpolate(x, scale_factor=2, mode="nearest")
        ph, pw = (pad, pad) if isinstance(pad, int) else pad
        if pad_mode == "reflect":
            x, ph, pw = F.pad(x, (pw, pw, ph, ph), mode="reflect"), 0, 0
        y = F.conv2d(x, w, b, stride=stride, padding=(ph, pw))
        if bn is not None:
            nrm = {k: self.sd[f"{bn}.{k}"] for k in ("weight", "bias", "running_mean", "running_var")}
            y = (y - nrm["running_mean"].view(1, -1, 1, 1)) / torch.sqrt(nrm["running_var"].view(1, -1, 1, 1) + 1e-5) * \
                nrm["weight"].view(1, -1, 1, 1) + nrm["bias"].view(1, -1, 1, 1)
        y = {"none": lambda t: t, "relu": torch.relu, "leaky": lambda t: F.leaky_relu(t, 0.2),
             "sigmoid": torch.sigmoid, "tanh": torch.tanh}[act](y) * scale
        return y if residual is None else y + residual.double()

    def lstm(self, name, xh, prev_cell):
        gates = F.conv2d(xh.double(), self.sd[name + ".weight"], self.sd[name + ".bias"], padding=1)
        i_g, r_g, o_g, c_g = gates.chunk(4, 1)
        cp = torch.zeros_like(i_g) if prev_cell is None else prev_cell.double()
        cell = torch.sigmoid(r_g) * cp + torch.sigmoid(i_g) * torch.tanh(c_g)
        return torch.sigmoid(o_g) * torch.tanh(cell), cell

    def maxpool(self, x):
        return F.max_pool2d(x.double(), 2, 2)

    def inorm(self, x, relu):
        y = F.instance_norm(x.double(), eps=1e-5)
        return torch.relu(y) if relu else y

    def add_relu(self, x, y):
        return torch.relu(x.double() + y.double())

    def gru_rh(self, r, h):
        return r.double() * h.double()

    def gru_mix(self, z, h, q):
        return (1 - z.double()) * h.double() + z.double() * q.double()

    def convex(self, flow, mask):
        return FO.convex_upsample(flow.double(), mask.double())


# ---------------------------------------------------------------------------------------------------------------
# Launch recorder (device side)
# ---------------------------------------------------------------------------------------------------------------
class Launch:
    def __init__(self, idx, kind, **kw):
        self.idx, self.kind = idx, kind
        self.__dict__.update(kw)
        self.taken = []                     # (lo, hi) output-row ranges matched so far

    def __repr__(self):
        return f"<launch {self.idx} {self.kind} {getattr(self, 'wname', '')}>"


def _chain_snapshot(ch):
    ph, pw = ch.desc.pad_h, ch.desc.pad_w
    return dict(snap=chain_view(ch, ch.n, ch.cin, ch.h, ch.w, (ph, pw)).clone(), cin=ch.cin, h=ch.h, w=ch.w,
                pad=(ph, pw), pad_mode=ch.pad_mode)


def _chain_block(ch, c_off, cout):
    ph, pw = ch.desc.pad_h, ch.desc.pad_w
    v = chain_view(ch, ch.n, ch.cin, ch.h, ch.w, (ph, pw))
    return v[:, ph:ph + ch.h, pw:pw + ch.w, c_off:c_off + cout].permute(0, 3, 1, 2).float().contiguous()


class Recorder:
    """Context manager: patches the `b200.nn` entry points the modules call (they look them up through `K.` at call
    time), runs each call, then snapshots its operands and outputs on the same stream before the next launch can reuse
    a chained buffer.  Calls made from inside another patched call (the fp32 path's explicit bilinear upsampling inside
    conv2d) are part of that launch.  `modules`: {prefix: nn.Module}; parameters are named prefix + named_parameters()."""

    def __init__(self, modules):
        from b200 import nn as K
        self.K = K
        self.modules = modules
        self.launches = []
        self._depth = 0
        self.pname = {}                              # id(parameter) -> name
        self.ptr_name = {}                           # data_ptr of a weight parameter -> module name
        self.mods = {}                               # module name -> module
        for prefix, m in modules.items():
            for n, t in m.named_parameters():
                self.pname[id(t)] = prefix + n
                if n.endswith(".weight"):
                    self.ptr_name[t.data_ptr()] = prefix + n[:-len(".weight")]
            for n, mod in m.named_modules():
                self.mods[prefix + n] = mod

    def resolve(self, w):
        """(how, [source module names]) of a weight tensor passed to a launch: 'param', 'merged' (torch.cat of the
        sources' weights along Cout), 'folded' (batch norm folded in) or 'input_half' (the ConvLSTM gates' x half)."""
        if id(w) in self.pname:
            return "param", [self.pname[id(w)][:-len(".weight")]]
        for name, mod in self.mods.items():
            if mod.__dict__.get("_w_in") is w:
                return "input_half", [name + ".Gates"]
            for key, ws, _ in mod.__dict__.get("_merged_cache", {}).values():
                if ws is w:
                    return "merged", [self.ptr_name[k[0]] for k in key]
        from src.models.stage_1.core import extractor
        for key, ws, _ in extractor._fold_cache.values():
            if ws is w:
                return "folded", [self.ptr_name[key[0][0]]]
        raise AssertionError(f"launch weight of shape {tuple(w.shape)} is no parameter, merge, fold or gate half")

    def __enter__(self):
        self._saved = {f: getattr(self.K, f) for f in FNS}
        for f in FNS:
            setattr(self.K, f, self._wrap(f, self._saved[f]))
        return self

    def __exit__(self, *exc):
        for f, fn in self._saved.items():
            setattr(self.K, f, fn)

    def _wrap(self, kind, orig):
        sig = inspect.signature(orig)

        def wrapper(*a, **kw):
            if self._depth:
                return orig(*a, **kw)
            ba = sig.bind(*a, **kw)
            ba.apply_defaults()
            args = dict(ba.arguments)
            self._depth += 1
            try:
                res = orig(*a, **kw)
            finally:
                self._depth -= 1
            self.launches.append(getattr(self, "_snap_" + kind, self._snap_plain)(len(self.launches), kind, args, res))
            return res
        return wrapper

    def _snap_conv2d(self, idx, kind, a, res):
        K = self.K
        x, w = a["x"], a["w"]
        cout = w.shape[0]
        how, srcs = self.resolve(w)
        rec = dict(how=how, srcs=srcs, wname=",".join(srcs), w=w, b=a["b"], stride=a["stride"],
                   pad=(a["pad"], a["pad"]) if isinstance(a["pad"], int) else tuple(a["pad"]), pad_mode=a["pad_mode"],
                   act=a["act"], upsample=a["upsample"], up_mode=a["upsample_mode"], scale=float(a["out_scale"]),
                   tc=(a["precision"] or K.conv_precision()) == "tc" or isinstance(x, K.Chain) or a["chain_out"] is not None)
        if isinstance(x, K.Chain):
            rec["chain"] = _chain_snapshot(x)
        else:
            lo, hi = a["in_slice"] or (0, x.shape[1])
            rec["operand"] = x[:, lo:hi].clone()
        r = a["residual"]
        rec["residual"] = None if r is None else r[:, a["res_c_off"]:a["res_c_off"] + cout].clone()
        rec["out"] = None if res is None else res[:, a["out_c_off"]:a["out_c_off"] + cout].clone()
        co = a["chain_out"]
        rec["chain_out"] = None if co is None else _chain_block(co, a["chain_c_off"], cout)
        return Launch(idx, kind, **rec)

    def _snap_convlstm(self, idx, kind, a, res):
        K = self.K
        x, w = a["x"], a["weight"]
        how, srcs = self.resolve(w)
        st = a["prev_state"]
        rec = dict(how=how, srcs=srcs, wname=srcs[0], w=w, b=a["bias"], tc=True,
                   prev_hidden=None if st is None else st[0].clone(), prev_cell=None if st is None else st[1].clone(),
                   hidden=res[0].clone(), cell=None if res[1] is None else res[1].clone())
        if isinstance(x, K.Chain):
            rec["chain"] = _chain_snapshot(x)
        else:
            rec["operand"] = x.clone() if st is None else torch.cat((x, st[0]), 1)
        return Launch(idx, kind, **rec)

    def _snap_convlstm_cell(self, idx, kind, a, res):
        return Launch(idx, kind, gates=a["gates"].clone(),
                      prev_cell=None if a["prev_cell"] is None else a["prev_cell"].clone(),
                      hidden=res[0].clone(), cell=None if res[1] is None else res[1].clone())

    def _snap_convlstm_zero_state(self, idx, kind, a, res):
        return Launch(idx, "convlstm_cell", gates=a["gates"].clone(), prev_cell=None, hidden=res[0].clone(),
                      cell=None if res[1] is None else res[1].clone())

    def _snap_gru_gate(self, idx, kind, a, res):
        n = a["a"].shape[0]
        per = a["a"].numel() // n
        out = res.view(n, -1)[:, :per].reshape(a["a"].shape).clone()
        return Launch(idx, kind, mode=a["mode"], a=a["a"].clone(), b=a["b"].clone(),
                      c=None if a["c"] is None else a["c"].clone(), out=out)

    def _snap_instance_norm(self, idx, kind, a, res):
        return Launch(idx, kind, x=a["x"].clone(), eps=a["eps"], relu=a["relu"], out=res.clone())

    def _snap_plain(self, idx, kind, a, res):
        return Launch(idx, kind, args={k: (v.clone() if isinstance(v, torch.Tensor) else v) for k, v in a.items()},
                      out=res.clone())


# ---------------------------------------------------------------------------------------------------------------
# Launch checker (device side)
# ---------------------------------------------------------------------------------------------------------------
def _bits(t):
    return t.contiguous().view(torch.int16 if t.dtype == torch.float16 else torch.int32)


def _check_chain(ch, want, what):
    """(a) for a chained operand: interior = rn_f16(satfinite(want)) bit for bit, halo zero or mirrored, channel padding
    zero.  Returns the interior as fp32 NCHW."""
    snap, cin, h, w, (ph, pw) = ch["snap"], ch["cin"], ch["h"], ch["w"], ch["pad"]
    assert tuple(want.shape[1:]) == (cin, h, w), f"{what}: chained operand shape {(cin, h, w)} != {tuple(want.shape)}"
    want16 = want.clamp(-65504.0, 65504.0).half().permute(0, 2, 3, 1)
    inner = snap[:, ph:ph + h, pw:pw + w, :cin]
    n_bad = int((_bits(inner) != _bits(want16)).sum())
    assert n_bad == 0, f"{what}: {n_bad} chained operand values differ from rn_f16 of the assembled input"
    assert not bool(_bits(snap[..., cin:]).any()), f"{what}: channel padding of the chained operand is not zero"
    if ch["pad_mode"] == "reflect":
        full = F.pad(inner.permute(0, 3, 1, 2).float(), (pw, pw, ph, ph), mode="reflect").half().permute(0, 2, 3, 1)
        n_bad = int((_bits(snap[..., :cin]) != _bits(full)).sum())
        assert n_bad == 0, f"{what}: {n_bad} halo values of the chained operand are not the reflection of the interior"
    else:
        halo = torch.ones(snap.shape[1:3], dtype=torch.bool, device=snap.device)
        halo[ph:ph + h, pw:pw + w] = False
        assert not bool(_bits(snap[:, halo]).any()), f"{what}: zero halo of the chained operand was written"
    return inner.permute(0, 3, 1, 2).float()


def _equal(got, want, what):
    assert got.shape == want.shape, f"{what}: shape {tuple(got.shape)} != {tuple(want.shape)}"
    n_bad = int((_bits(got.float()) != _bits(want.float())).sum())
    assert n_bad == 0, f"{what}: {n_bad} of {got.numel()} values differ"


class LaunchChecker(_Deps):
    """Matches the dataflow's layers with the recorded launches and checks them (module docstring).  `params`:
    {name: tensor} of the recorded modules with their prefixes, buffers included; `ratios` collects the largest
    error / bound per label."""

    def __init__(self, rec, params, label, ratios):
        super().__init__()
        self.rec, self.params, self.label, self.ratios = rec, params, label, ratios
        self.by_name = {}
        for L in rec.launches:
            for s in getattr(L, "srcs", ()):
                self.by_name.setdefault(s, []).append(L)
        self.next_of_kind = {}

    def _ratio(self, what, r):
        key = self.label
        self.ratios[key] = max(self.ratios.get(key, 0.0), r)

    def _take(self, name):
        ls = self.by_name.get(name)
        assert ls, f"no launch uses the parameters of {name}"
        L = ls.pop(0)
        lo = 0
        for s in L.srcs:
            rows = self.params[s + ".weight"].shape[0]
            if s == name:
                break
            lo += rows
        hi = lo + self.params[name + ".weight"].shape[0]
        if L.how == "input_half":
            lo, hi = 0, L.w.shape[0]
        assert (lo, hi) not in L.taken, f"{name}: launch {L} matched twice"
        L.taken.append((lo, hi))
        return L, lo, hi

    def _take_kind(self, kind, deps):
        i = self.next_of_kind.get(kind, 0)
        ls = [L for L in self.rec.launches if L.kind == kind]
        assert i < len(ls), f"no {kind} launch left"
        self.next_of_kind[kind] = i + 1
        L = ls[i]
        L.taken.append((0, 0))
        assert L.idx > deps, f"{L} runs before a launch it depends on ({deps})"
        return L

    def conv(self, name, x, stride=1, pad=0, pad_mode="zeros", act="none", up=None, scale=1.0, residual=None, bn=None):
        L, lo, hi = self._take(name)
        what = f"{self.label} {name} (launch {L.idx})"
        assert L.kind == "conv2d", what
        assert L.idx > self.dep(x, residual), f"{what} runs before a launch it depends on"
        pad = (pad, pad) if isinstance(pad, int) else tuple(pad)
        assert (L.stride, L.pad, L.pad_mode, L.act, L.scale) == (stride, pad, pad_mode, act, scale), \
            f"{what}: launch geometry {(L.stride, L.pad, L.pad_mode, L.act, L.scale)}"
        assert (L.upsample, L.up_mode if L.upsample == 2 else None) == ((2, up) if up else (1, None)), what
        # c. host-built weights
        W, B = self.params[name + ".weight"], self.params.get(name + ".bias")
        w_l, b_l = L.w[lo:hi].detach(), None if L.b is None else L.b[lo:hi].detach()
        if L.how == "folded":
            nrm = {k: self.params[f"{bn}.{k}"] for k in ("weight", "bias", "running_mean", "running_var")}
            w64, b64, s = _bn_fold64(nrm, W, B)
            ew, eb = 5 * U * w64.abs(), 6 * U * ((B.double() - nrm["running_mean"].double()) * s).abs() + 2 * U * b64.abs()
            rw = float(((w_l.double() - w64).abs() / ew.clamp_min(1e-300)).max())
            rb = float(((b_l.double() - b64).abs() / eb.clamp_min(1e-300)).max())
            assert rw <= 1 and rb <= 1, f"{what}: folded weight / bias off the float64 fold by {rw:.2f} / {rb:.2f} bounds"
        else:
            assert bn is None, f"{what}: batch norm is not folded into the launch"
            if L.how == "input_half":
                _equal(w_l, W[:, :w_l.shape[1]], what + " gate input half")
            else:
                _equal(w_l, W, what + " weight")
            assert (b_l is None) == (B is None), what
            if B is not None:
                _equal(b_l, B, what + " bias")
        # a. operands
        cin = L.w.shape[1]
        if L.how == "input_half":
            assert not bool(x[:, cin:].any()), f"{what}: the gates' input half is used with a nonzero hidden state"
            x = x[:, :cin]
        if "chain" in L.__dict__:
            opnd = _check_chain(L.chain, x, what)
        else:
            _equal(L.operand, x, what + " operand")
            opnd = L.operand
        assert (L.residual is None) == (residual is None), what
        if residual is not None:
            _equal(L.residual, residual, what + " residual")
        # b. the launch against float64 on its own operands, one sample at a time (device memory)
        y = L.out[:, lo:hi] if L.out is not None else L.chain_out[:, lo:hi]
        n, _, h, w = opnd.shape
        c = dict(n=1, cin=cin, h=h, w=w, cout=hi - lo, k=tuple(w_l.shape[2:]), stride=stride, pad=pad,
                 pad_mode=pad_mode, act=act, upsample=2 if up else 1, up_mode=up or "nearest", in_slice=None,
                 res_slice=None if residual is None else (0, hi - lo), out_scale=scale)
        ratio, bad, err = 0.0, 0, 0.0
        for i in range(n):
            yi = y[i:i + 1]
            y_ref, slack, unit = reference(c, opnd[i:i + 1], w_l, b_l,
                                           None if L.residual is None else L.residual[i:i + 1], L.tc)
            if L.out is None:               # stored only as fp16 into a chain: one more rounding
                slack = slack + 2.0 ** -11 * yi.double().abs() + 2.0 ** -25
            r_i, bad_i, err_i = bound_ratio(yi, y_ref, slack, unit, C_TC if L.tc else C_FP32)
            ratio, bad, err = max(ratio, r_i), bad + bad_i, max(err, err_i)
            del y_ref, slack, unit
        self._ratio(what, ratio)
        assert bool(torch.isfinite(y).all()), f"{what}: non-finite output"
        assert not bad, f"{what}: {bad} elements beyond the bound (ratio {ratio:.3f}, max err {err:.3e})"
        if L.chain_out is not None and L.out is not None:
            _equal(L.chain_out[:, lo:hi], y.clamp(-65504.0, 65504.0).half().float(), what + " chained copy")
        return self.mark(y, L.idx)

    def lstm(self, name, xh, prev_cell):
        deps = self.dep(xh, prev_cell)
        L, _, _ = self._take(name)
        what = f"{self.label} {name} (launch {L.idx})"
        c = self.params[name + ".weight"].shape[0] // 4
        if L.kind == "conv2d":                # fp32 path: the gate convolution, then the cell kernel
            self.by_name[name].insert(0, L)
            L.taken.pop()
            gates = self.conv(name, xh, pad=1)
            C = self._take_kind("convlstm_cell", self.dep(gates, prev_cell))
            _equal(C.gates, gates, what + " cell kernel gates")
            assert (C.prev_cell is None) == (prev_cell is None), what
            if prev_cell is not None:
                _equal(C.prev_cell, prev_cell, what + " previous cell")
            hid, cell, e_h, e_c = cell_reference(C.gates.double(), torch.zeros_like(C.gates, dtype=torch.float64),
                                                 C.prev_cell)
            idx = C.idx
        else:
            assert L.kind == "convlstm" and L.idx > deps, what
            assert (L.prev_cell is None) == (prev_cell is None), what
            if L.how == "input_half":
                _equal(L.w, self.params[name + ".weight"][:, :L.w.shape[1]], what + " gate input half")
                assert not bool(xh[:, c:].any()), f"{what}: zero-state launch with a nonzero hidden state"
                want = xh[:, :c]
            else:
                _equal(L.w, self.params[name + ".weight"], what + " weight")
                _equal(L.prev_hidden, xh[:, c:], what + " previous hidden state")
                _equal(L.prev_cell, prev_cell, what + " previous cell")
                want = xh
            _equal(L.b, self.params[name + ".bias"], what + " bias")
            if "chain" in L.__dict__:
                opnd = _check_chain(L.chain, want, what)
            else:
                _equal(L.operand, want, what + " operand")
                opnd = L.operand
            hid, cell, e_h, e_c = convlstm_reference(opnd, L.w.detach(), L.b.detach(), L.prev_cell)
            C, idx = L, L.idx
        for part, got, ref, e in (("hidden", C.hidden, hid, e_h), ("cell", C.cell, cell, e_c)):
            err = (got.double() - ref).abs()
            r = float((err / e.clamp_min(1e-300)).max())
            self._ratio(f"{what} {part}", r)
            assert r <= 1.0, f"{what} {part}: error / bound {r:.3f}"
        return self.mark(C.hidden, idx), self.mark(C.cell, idx)

    def maxpool(self, x):
        L = self._take_kind("maxpool2", self.dep(x))
        what = f"{self.label} maxpool2 (launch {L.idx})"
        _equal(L.args["x"], x, what + " operand")
        _equal(L.out, F.max_pool2d(L.args["x"], 2, 2), what)
        return self.mark(L.out, L.idx)

    def inorm(self, x, relu):
        L = self._take_kind("instance_norm", self.dep(x))
        what = f"{self.label} instance_norm (launch {L.idx})"
        assert L.relu == relu and L.eps == 1e-5, what
        _equal(L.x, x, what + " operand")
        xd = L.x.double()
        mean = xd.mean(dim=(2, 3), keepdim=True)
        var = ((xd - mean) ** 2).mean(dim=(2, 3), keepdim=True)
        ref = (xd - mean) / torch.sqrt(var + 1e-5)
        if relu:
            ref = torch.relu(ref)
        scale = (mean.abs() / var.sqrt().clamp_min(1e-30)).amax(dim=(2, 3)).clamp_max(1e3) + ref.abs().amax(dim=(2, 3)) + 1
        r = float(((L.out.double() - ref).abs().amax(dim=(2, 3)) / (6 * U * scale)).max())
        self._ratio(what, r)
        assert r <= 1.0, f"{what}: error / bound {r:.3f}"
        return self.mark(L.out, L.idx)

    def add_relu(self, x, y):
        L = self._take_kind("add_relu", self.dep(x, y))
        what = f"{self.label} add_relu (launch {L.idx})"
        _equal(L.args["a"], x, what + " shortcut")
        _equal(L.args["b"], y, what + " block output")
        _equal(L.out, torch.relu(L.args["a"] + L.args["b"]), what)
        return self.mark(L.out, L.idx)

    def gru_rh(self, r, h):
        L = self._take_kind("gru_gate", self.dep(r, h))
        what = f"{self.label} gru_gate r*h (launch {L.idx})"
        assert L.mode == 0, what
        _equal(L.a, r, what + " r")
        _equal(L.b, h, what + " h")
        _equal(L.out, L.a * L.b, what)
        return self.mark(L.out, L.idx)

    def gru_mix(self, z, h, q):
        L = self._take_kind("gru_gate", self.dep(z, h, q))
        what = f"{self.label} gru_gate (1-z)h+zq (launch {L.idx})"
        assert L.mode == 1, what
        _equal(L.a, z, what + " z")
        _equal(L.b, h, what + " h")
        _equal(L.c, q, what + " q")
        a, b, c = L.a.double(), L.b.double(), L.c.double()
        r = float(((L.out.double() - ((1 - a) * b + a * c)).abs() / (4 * U * (b.abs() + c.abs())).clamp_min(1e-300)).max())
        self._ratio(what, r)
        assert r <= 1.0, f"{what}: error / bound {r:.3f}"
        return self.mark(L.out, L.idx)

    def convex(self, flow, mask):
        L = self._take_kind("convex_upsample", self.dep(flow, mask))
        what = f"{self.label} convex_upsample (launch {L.idx})"
        _equal(L.args["flow"], flow, what + " flow")
        _equal(L.args["mask"], mask, what + " mask")
        ref = FO.convex_upsample(L.args["flow"].double(), L.args["mask"].double())
        bound = 8 * U * 8 * float(L.args["flow"].abs().max())
        r = float((L.out.double() - ref).abs().max()) / bound
        self._ratio(what, r)
        assert r <= 1.0, f"{what}: error / bound {r:.3f}"
        return self.mark(L.out, L.idx)

    def finish(self):
        """(d): every launch matched exactly once, a merged one by row ranges that tile its output channels."""
        for L in self.rec.launches:
            if L.kind in ("conv2d", "convlstm") and L.how == "merged":
                rows = sorted(L.taken)
                assert rows and rows[0][0] == 0 and rows[-1][1] == L.w.shape[0] and \
                    all(a[1] == b[0] for a, b in zip(rows, rows[1:])), f"{self.label}: merged {L} rows {rows}"
            else:
                assert len(L.taken) == 1, f"{self.label}: {L} matched {len(L.taken)} times"


def params_of(modules):
    """{prefix + name: tensor} of the modules' parameters and buffers (what LaunchChecker and ExactDevice read)."""
    out = {}
    for prefix, m in modules.items():
        for n, t in m.state_dict(keep_vars=True).items():
            out[prefix + n] = t.detach()
    return out


def max_abs_rel(a, b):
    return float((a.double() - b.double()).abs().max()) / max(float(b.double().abs().max()), 1e-300)

