"""RAFT update operator with the reference's module tree / state_dict keys
(src/models/stage_1/core/update.py:6-136): BasicMotionEncoder, SepConvGRU, FlowHead, mask head.
Parameters live in nn.Conv2d modules (for checkpoints); arithmetic runs in b200_conv2d / b200_gru_gate.
The reference runs this block under fp16 autocast; the convolution arithmetic here follows
b200.nn.conv_precision() (RAFT.forward selects the wgmma fp16-operand path when args.mixed_precision)."""
import torch
import torch.nn as nn

from b200 import nn as K


def _c(conv, x, act="none", **kw):
    return K.conv2d(x, conv.weight, conv.bias.detach() if conv.bias is not None else None,
                    pad=conv.padding, act=act, **kw)


def _merged(owner, name, convs):
    """Weights / biases of convolutions that read the SAME input with the same geometry and activation, stacked
    along Cout so that they run as one launch (each output channel is still its own dot product: results are
    unchanged).  Cached on the module, rebuilt when a source parameter is replaced or modified in place."""
    key = tuple((c.weight.data_ptr(), c.weight._version, c.bias.data_ptr(), c.bias._version) for c in convs)
    cache = owner.__dict__.setdefault("_merged_cache", {})
    ent = cache.get(name)
    if ent is None or ent[0] != key:
        ent = (key, torch.cat([c.weight.detach() for c in convs], 0).contiguous(),
               torch.cat([c.bias.detach() for c in convs], 0).contiguous())
        cache[name] = ent
    return ent[1], ent[2]


class FlowHead(nn.Module):
    def __init__(self, input_dim=128, hidden_dim=256):
        super().__init__()
        self.conv1 = nn.Conv2d(input_dim, hidden_dim, 3, padding=1)
        self.conv2 = nn.Conv2d(hidden_dim, 2, 3, padding=1)

    def forward(self, x):
        return _c(self.conv2, _c(self.conv1, x, "relu"))


class SepConvGRU(nn.Module):
    def __init__(self, hidden_dim=128, input_dim=192 + 128):
        super().__init__()
        for tag, k, p in (("1", (1, 5), (0, 2)), ("2", (5, 1), (2, 0))):
            for g in "zrq":
                setattr(self, f"conv{g}{tag}", nn.Conv2d(hidden_dim + input_dim, hidden_dim, k, padding=p))
        self.hidden_dim = hidden_dim

    def forward(self, h, x):
        n, c, hh, ww = h.shape
        hx = torch.empty(n, c + x.shape[1], hh, ww, dtype=torch.float32, device=h.device)
        hx[:, c:] = x                                           # the x half of both concats never changes
        for tag in ("1", "2"):
            hx[:, :c] = h
            cz, cr = getattr(self, "convz" + tag), getattr(self, "convr" + tag)
            w, b = _merged(self, "zr" + tag, (cz, cr))          # z and r gates: one convolution, Cout = 2c
            zr = K.conv2d(hx, w, b, pad=cz.padding, act="sigmoid")
            z, r = zr[:, :c].contiguous(), zr[:, c:].contiguous()   # views for batch 1
            K.gru_gate(r, h, out=hx, mode=0)                    # [r*h, x]
            q = _c(getattr(self, "convq" + tag), hx, "tanh")
            h = K.gru_gate(z, h, q, mode=1)                     # (1-z)*h + z*q
        return h


class BasicMotionEncoder(nn.Module):
    def __init__(self, args):
        super().__init__()
        cor_planes = args.corr_levels * (2 * args.corr_radius + 1) ** 2
        self.convc1 = nn.Conv2d(cor_planes, 256, 1, padding=0)
        self.convc2 = nn.Conv2d(256, 192, 3, padding=1)
        self.convf1 = nn.Conv2d(2, 128, 7, padding=3)
        self.convf2 = nn.Conv2d(128, 64, 3, padding=1)
        self.conv = nn.Conv2d(64 + 192, 128 - 2, 3, padding=1)

    def forward(self, flow, corr):
        n, _, h, w = flow.shape
        if K.Chain.available():
            # wgmma path: each convolution's epilogue writes the packed fp16 input of the next one (the 192 + 64
            # channel concat included) — three fp32 intermediates and three repack kernels less per iteration
            dev = flow.device
            c2 = K.Chain(n, 256, h, w, (3, 3), 1, dev, tag="convc2")
            _c(self.convc1, corr, "relu", chain_out=c2, keep_fp32=False)
            f2 = K.Chain(n, 128, h, w, (3, 3), 1, dev, tag="convf2")
            _c(self.convf1, flow, "relu", chain_out=f2, keep_fp32=False)
            cf = K.Chain(n, 256, h, w, (3, 3), 1, dev, tag="cor_flo")
            _c(self.convc2, c2, "relu", chain_out=cf, chain_c_off=0, keep_fp32=False)
            _c(self.convf2, f2, "relu", chain_out=cf, chain_c_off=192, keep_fp32=False)
            out = torch.empty(n, 128, h, w, dtype=torch.float32, device=dev)
            _c(self.conv, cf, "relu", out=out, out_c_off=0)
            out[:, 126:] = flow
            return out
        cor_flo = torch.empty(n, 256, h, w, dtype=torch.float32, device=flow.device)
        _c(self.convc2, _c(self.convc1, corr, "relu"), "relu", out=cor_flo, out_c_off=0)
        _c(self.convf2, _c(self.convf1, flow, "relu"), "relu", out=cor_flo, out_c_off=192)
        out = torch.empty(n, 128, h, w, dtype=torch.float32, device=flow.device)
        _c(self.conv, cor_flo, "relu", out=out, out_c_off=0)
        out[:, 126:] = flow
        return out


class BasicUpdateBlock(nn.Module):
    def __init__(self, args, hidden_dim=128, input_dim=128):
        super().__init__()
        self.args = args
        self.encoder = BasicMotionEncoder(args)
        self.gru = SepConvGRU(hidden_dim=hidden_dim, input_dim=128 + hidden_dim)
        self.flow_head = FlowHead(hidden_dim, hidden_dim=256)
        self.mask = nn.Sequential(nn.Conv2d(128, 256, 3, padding=1), nn.ReLU(inplace=True),
                                  nn.Conv2d(256, 64 * 9, 1, padding=0))

    def forward(self, net, inp, corr, flow, upsample=True):
        motion = self.encoder(flow, corr)
        net = self.gru(net, torch.cat([inp, motion], dim=1))
        # flow head and mask head both start with a 3x3 128->256 ReLU convolution of `net`: one launch, Cout = 512
        w, b = _merged(self, "heads", (self.flow_head.conv1, self.mask[0]))
        hm = K.conv2d(net, w, b, pad=self.mask[0].padding, act="relu")
        delta_flow = _c(self.flow_head.conv2, hm, in_slice=(0, 256))
        mask = _c(self.mask[2], hm, in_slice=(256, 512), out_scale=0.25)           # .25 * mask head
        return net, mask, delta_flow
