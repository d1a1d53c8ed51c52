"""`TransformNet` local refinement (Lai et al.) with the reference's constructor, state_dict keys and call
signature (src/models/network_local.py:7-188): `forward(X, prev_state)` returns `(Y, (hidden, cell))`, and the
returned state (fresh tensors) can be passed back as the next frame's `prev_state`, the recurrent form of the
network; `None` is the zero state.  Reflection padding, nearest upsampling, LeakyReLU and the residual adds are
fused into the convolutions; on the wgmma path the ConvLSTM cell update runs in the gate convolution's epilogue
(b200_convlstm_tma), on the fp32 path in b200_convlstm_cell after the gate convolution.  As in the reference
the norm layers are constructed (their buffers are part of the state_dict) but never applied
(`self.norm in ["BN" or "IN"]`, network_local.py:136,169)."""
import torch
import torch.nn as nn

from b200 import nn as K


class ConvLayer(nn.Module):
    def __init__(self, in_channels, out_channels, kernel_size, stride, norm=None, bias=True):
        super().__init__()
        self.reflection_pad = nn.ReflectionPad2d(kernel_size // 2)
        self.conv2d = nn.Conv2d(in_channels, out_channels, kernel_size, stride, bias=bias)
        self.norm = norm
        if norm == "BN":
            self.norm_layer = nn.BatchNorm2d(out_channels)
        elif norm == "IN":
            self.norm_layer = nn.InstanceNorm2d(out_channels, track_running_stats=True)
        self.upsample = None

    def run(self, x, act="none", **kw):
        if self.norm == "BN":
            raise NotImplementedError("norm='BN' (the only value for which the reference applies a norm) is unused")
        c = self.conv2d
        return K.conv2d(x, c.weight, c.bias.detach() if c.bias is not None else None, stride=c.stride[0],
                        pad=c.kernel_size[0] // 2, pad_mode="reflect", act=act, upsample=self.upsample or 1, **kw)


class UpsampleConvLayer(ConvLayer):
    def __init__(self, in_channels, out_channels, kernel_size, stride, upsample=None, norm=None, bias=True):
        super().__init__(in_channels, out_channels, kernel_size, stride, norm=norm, bias=bias)
        self.upsample = upsample
        if upsample:
            self.upsample_layer = nn.Upsample(scale_factor=upsample, mode='nearest')


class ResidualBlock(nn.Module):
    def __init__(self, channels, norm=None, bias=True):
        super().__init__()
        self.conv1 = ConvLayer(channels, channels, kernel_size=3, stride=1, bias=bias, norm=norm)
        self.conv2 = ConvLayer(channels, channels, kernel_size=3, stride=1, bias=bias, norm=norm)

    def run(self, x):
        return self.conv2.run(self.conv1.run(x, "leaky"), residual=x)

    def run_chained(self, x_chain, x, next_chain, tag):
        """wgmma path: `x_chain` is this block's packed input (written by the previous convolution), `x` the same
        tensor in fp32 (the residual); conv1's output exists only as conv2's packed input; conv2's output is written in
        fp32 (next residual) and into `next_chain` (the packed input of the next convolution)."""
        n, c, h, w = x.shape
        mid = K.Chain(n, c, h, w, (3, 3), 1, x.device, tag=tag, pad_mode="reflect")
        self.conv1.run(x_chain, "leaky", chain_out=mid, keep_fp32=False)
        return self.conv2.run(mid, residual=x, chain_out=next_chain)


class ConvLSTM(nn.Module):
    def __init__(self, input_size, hidden_size, kernel_size):
        super().__init__()
        self.input_size, self.hidden_size = input_size, hidden_size
        self.Gates = nn.Conv2d(input_size + hidden_size, 4 * hidden_size, kernel_size, padding=kernel_size // 2)

    def run(self, x, prev_state=None):
        """One step -> fresh (hidden, cell) tensors.  `x` is a tensor, or on the wgmma path a `Chain` (input_size
        channels without a state, input_size + hidden_size with one: the previous hidden state is packed behind x).
        wgmma path: the gate convolution with the cell update in its epilogue (K.convlstm); fp32 path: the gate
        convolution on cat(x, prev_hidden), then the cell kernel."""
        gw, gb = self.Gates.weight, self.Gates.bias.detach()
        tc = isinstance(x, K.Chain) or K.Chain.available()
        if prev_state is None:
            # zero previous hidden state: only the input half of the gate weights contributes
            if getattr(self, "_w_in_key", None) != (gw.data_ptr(), gw._version):       # input half, sliced once
                self._w_in = gw.detach()[:, :self.input_size].contiguous()
                self._w_in_key = (gw.data_ptr(), gw._version)
            if tc:
                return K.convlstm(x, self._w_in, gb)
            gates = K.conv2d(x, self._w_in, gb, pad=self.Gates.padding)
            return K.convlstm_zero_state(gates)
        if tc:
            return K.convlstm(x, gw, gb, prev_state)
        n, _, h, w = x.shape
        hidden, cell = K._check_state(prev_state, (n, self.hidden_size, h, w), x.device)
        gates = K.conv2d(torch.cat((x, hidden), 1), gw, gb, pad=self.Gates.padding)
        return K.convlstm_cell(gates, cell)


class TransformNet(nn.Module):
    def __init__(self, opts, nc_in, nc_out):
        super().__init__()
        self.blocks, self.epoch = opts.blocks, 0
        nf, norm = opts.nf, opts.norm
        use_bias = (norm == "IN")
        self.conv1a = ConvLayer(3 + 3, nf, kernel_size=7, stride=1, bias=use_bias, norm=norm)
        self.conv1b = ConvLayer(3 + 3, nf, kernel_size=7, stride=1, bias=use_bias, norm=norm)
        self.conv2a = ConvLayer(nf, nf * 2, kernel_size=3, stride=2, bias=use_bias, norm=norm)
        self.conv2b = ConvLayer(nf, nf * 2, kernel_size=3, stride=2, bias=use_bias, norm=norm)
        self.conv3 = ConvLayer(nf * 4, nf * 4, kernel_size=3, stride=2, bias=use_bias, norm=norm)
        self.ResBlocks = nn.ModuleList(ResidualBlock(nf * 4, bias=use_bias, norm=norm) for _ in range(self.blocks))
        self.convlstm = ConvLSTM(input_size=nf * 4, hidden_size=nf * 4, kernel_size=3)
        self.deconv1 = UpsampleConvLayer(nf * 4, nf * 2, kernel_size=3, stride=1, upsample=2, bias=use_bias, norm=norm)
        self.deconv2 = UpsampleConvLayer(nf * 4, nf, kernel_size=3, stride=1, upsample=2, bias=use_bias, norm=norm)
        self.deconv3 = ConvLayer(nf * 2, nc_out, kernel_size=7, stride=1)
        self.nf = nf

    @torch.no_grad()
    def forward(self, X, prev_state):
        X = X.float().contiguous()
        n, _, h, w = X.shape
        nf, dev = self.nf, X.device
        c1 = torch.empty(n, 2 * nf, h, w, dtype=torch.float32, device=dev)          # [D1 | E1a]
        c2 = torch.empty(n, 4 * nf, h // 2, w // 2, dtype=torch.float32, device=dev)  # [D2 | E2a]
        e2 = torch.empty(n, 4 * nf, h // 2, w // 2, dtype=torch.float32, device=dev)  # [E2a | E2b]
        chained = K.Chain.available()
        # wgmma path: the last convolution's input [D1 | E1a] (64 channels at full resolution, the largest repack of the
        # network) is filled by the epilogues of deconv2 and conv1a
        c1_chain = K.Chain(n, 2 * nf, h, w, (7, 7), 3, dev, tag="tn_c1", pad_mode="reflect") if chained else None
        self.conv1a.run(X, "leaky", in_slice=(0, 6), out=c1, out_c_off=nf, chain_out=c1_chain, chain_c_off=nf)
        e1b = self.conv1b.run(X, "leaky", in_slice=(6, 12))
        self.conv2a.run(c1, "leaky", in_slice=(nf, 2 * nf), out=e2, out_c_off=0)
        self.conv2b.run(e1b, "leaky", out=e2, out_c_off=2 * nf)
        c2[:, 2 * nf:] = e2[:, :2 * nf]
        if chained:
            # wgmma path: conv3 -> 5 residual blocks -> ConvLSTM gates run as one chain of packed fp16 inputs (the
            # residuals stay fp32 tensors); eleven fp32 -> fp16 repack kernels less.  With a state the gates' input is
            # [RB | prev_hidden]: the last block writes channels [0, 4nf), the ConvLSTM packs the hidden state behind
            hq, wq = (h // 4, w // 4)
            chains = [K.Chain(n, 4 * nf, hq, wq, (3, 3), 1, dev, tag=f"tn_rb{i & 1}", pad_mode="reflect")
                      for i in range(len(self.ResBlocks))]
            gates_in = (K.Chain(n, 4 * nf, hq, wq, (3, 3), 1, dev, tag="tn_gates") if prev_state is None  # zero padding
                        else K.Chain(n, 8 * nf, hq, wq, (3, 3), 1, dev, tag="tn_gates_state"))        # (nn.Conv2d)
            rb = self.conv3.run(e2, "leaky", chain_out=chains[0] if chains else gates_in)
            for i, blk in enumerate(self.ResBlocks):
                nxt = chains[i + 1] if i + 1 < len(chains) else gates_in
                rb = blk.run_chained(chains[i], rb, nxt, tag="tn_mid")
            hidden, cell = self.convlstm.run(gates_in, prev_state)
        else:
            rb = self.conv3.run(e2, "leaky")
            for blk in self.ResBlocks:
                rb = blk.run(rb)
            hidden, cell = self.convlstm.run(rb, prev_state)
        self.deconv1.run(hidden, "leaky", out=c2, out_c_off=0)
        if chained:
            self.deconv2.run(c2, "leaky", chain_out=c1_chain, chain_c_off=0, keep_fp32=False)
            y = self.deconv3.run(c1_chain, "tanh")
        else:
            self.deconv2.run(c2, "leaky", out=c1, out_c_off=0)
            y = self.deconv3.run(c1, "tanh")
        return y, (hidden, cell)
