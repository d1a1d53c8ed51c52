"""`UNet` neural filter with the reference's constructor and state_dict keys
(src/models/network_filter.py:8-107); inference runs in b200_conv2d / b200_maxpool2 /
b200_upsample_bilinear2, skip concatenations are written in place (no torch.cat)."""
from collections import OrderedDict

import torch
import torch.nn as nn

from b200 import nn as K


class UNet(nn.Module):
    def __init__(self, in_channels=3, out_channels=1, init_features=32):
        super().__init__()
        f = init_features
        self.encoder1 = UNet._block(in_channels, f, "enc1")
        self.encoder2 = UNet._block(f, f * 2, "enc2")
        self.encoder3 = UNet._block(f * 2, f * 4, "enc3")
        self.encoder4 = UNet._block(f * 4, f * 8, "enc4")
        self.bottleneck = UNet._block(f * 8, f * 16, "bottleneck")
        for i, (cin, cout) in zip((4, 3, 2, 1), ((f * 16, f * 8), (f * 8, f * 4), (f * 4, f * 2), (f * 2, f))):
            setattr(self, f"upconv{i}", nn.Sequential(nn.Upsample(scale_factor=2, mode='bilinear', align_corners=True),
                                                      nn.Conv2d(cin, cout, kernel_size=3, padding=1)))
            setattr(self, f"decoder{i}", UNet._block(cout * 2, cout, f"dec{i}"))
        self.conv = nn.Conv2d(f, out_channels, kernel_size=1)

    @staticmethod
    def _block(cin, feat, name):
        return nn.Sequential(OrderedDict([(name + "conv1", nn.Conv2d(cin, feat, 3, padding=1, bias=False)),
                                          (name + "relu1", nn.ReLU(inplace=True)),
                                          (name + "conv2", nn.Conv2d(feat, feat, 3, padding=1, bias=False)),
                                          (name + "relu2", nn.ReLU(inplace=True))]))

    @staticmethod
    def _run_block(block, x, out=None, out_c_off=0, chain_out=None, chain_c_off=0, keep_fp32=True):
        convs = [m for m in block if isinstance(m, nn.Conv2d)]
        if K.Chain.available():
            # wgmma path: conv1's epilogue writes conv2's packed fp16 input directly — the intermediate tensor is
            # never written in fp32 nor repacked.  `x` may itself be a chained input, and conv2 may feed a chain.
            n, h, w = (x.n, x.h, x.w) if isinstance(x, K.Chain) else (x.shape[0], x.shape[2], x.shape[3])
            dev = x.buf.device if isinstance(x, K.Chain) else x.device
            ch = K.Chain(n, convs[1].in_channels, h, w, (3, 3), 1, dev)
            K.conv2d(x, convs[0].weight, None, pad=1, act="relu", chain_out=ch, keep_fp32=False)
            return K.conv2d(ch, convs[1].weight, None, pad=1, act="relu", out=out, out_c_off=out_c_off, chain_out=chain_out,
                            chain_c_off=chain_c_off, keep_fp32=keep_fp32)
        t = K.conv2d(x, convs[0].weight, None, pad=1, act="relu")
        return K.conv2d(t, convs[1].weight, None, pad=1, act="relu", out=out, out_c_off=out_c_off)

    @torch.no_grad()
    def forward(self, x):
        x = x.float().contiguous()
        n, _, h, w = x.shape
        dev = x.device
        cur = x
        if K.Chain.available():
            # wgmma path: the skip concatenations [upconv | encoder] exist only as the packed fp16 inputs of the decoder
            # blocks, filled by the epilogues of the two convolutions that produce them
            dec_in = []
            for i, enc in enumerate((self.encoder1, self.encoder2, self.encoder3, self.encoder4)):
                c = enc[0].out_channels
                ch = K.Chain(n, 2 * c, h >> i, w >> i, (3, 3), 1, dev, tag=f"unet_dec{i + 1}")
                e = UNet._run_block(enc, cur, chain_out=ch, chain_c_off=c)      # fp32 copy only for the pooling
                dec_in.append(ch)
                cur = K.maxpool2(e)
            cur = UNet._run_block(self.bottleneck, cur)
            last = K.Chain(n, self.conv.in_channels, h, w, (1, 1), 0, dev, tag="unet_out")     # input of the final 1x1
            for i, ch in zip((4, 3, 2, 1), reversed(dec_in)):
                up = getattr(self, f"upconv{i}")[1]
                K.conv2d(cur, up.weight, up.bias.detach(), pad=1, upsample=2, upsample_mode="bilinear", chain_out=ch,
                         chain_c_off=0, keep_fp32=False)
                if i == 1:
                    UNet._run_block(self.decoder1, ch, chain_out=last, keep_fp32=False)
                else:
                    cur = UNet._run_block(getattr(self, f"decoder{i}"), ch)
            return K.conv2d(last, self.conv.weight, self.conv.bias.detach())
        cats = []
        for i, enc in enumerate((self.encoder1, self.encoder2, self.encoder3, self.encoder4)):
            c = enc[0].out_channels
            hh, ww = h >> i, w >> i
            cat = torch.empty(n, 2 * c, hh, ww, dtype=torch.float32, device=dev)   # [upconv | encoder] (dim=1 cat)
            UNet._run_block(enc, cur, out=cat, out_c_off=c)
            cats.append(cat)
            cur = K.maxpool2(cat.narrow(1, c, c).contiguous())     # pool the encoder half of the concat buffer
        cur = UNet._run_block(self.bottleneck, cur)
        for i, cat in zip((4, 3, 2, 1), reversed(cats)):
            up = getattr(self, f"upconv{i}")[1]
            K.conv2d(cur, up.weight, up.bias.detach(), pad=1, out=cat, out_c_off=0, upsample=2,
                     upsample_mode="bilinear")
            cur = UNet._run_block(getattr(self, f"decoder{i}"), cat)
        return K.conv2d(cur, self.conv.weight, self.conv.bias.detach())
