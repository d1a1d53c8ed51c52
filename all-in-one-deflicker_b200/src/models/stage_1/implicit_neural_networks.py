"""`IMLP` with the reference's constructor / state_dict surface, evaluated by libb200deflicker.so.

Mirrors src/models/stage_1/implicit_neural_networks.py:15-81 of the reference: same ctor arguments,
parameters named ``hidden.{i}.weight|bias`` in nn.Linear layout and initialised from the global CPU
generator in the same order, ``forward(x: (rows, input_dim)) -> (rows, output_dim)`` with autograd.
All arithmetic (positional encoding, Linear stack, ReLU, skip concat, tanh and their gradients) runs
in the library's CUDA kernels through `b200_mlp_forward` / `b200_mlp_backward`; there is no PyTorch
fallback — calling it with CPU tensors raises.
"""
import ctypes as C
import math

import torch
import torch.nn as nn

from b200 import _native as N
from b200 import atlas as A


def count_parameters(model):
    return sum(p.numel() for p in model.parameters() if p.requires_grad)


class _ImlpFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, flat, module):
        if not x.is_cuda:
            raise N.B200Error("IMLP runs on CUDA tensors only (no CPU fallback)")
        lib = N.lib()
        x = x.contiguous().float()
        rows = x.shape[0]
        desc = module._desc
        enc = 2 * desc.input_dim * desc.pe_freqs if desc.pe_freqs > 0 else 0
        nbytes = int(lib.b200_mlp_workspace_bytes(C.byref(desc), rows, 1)) + rows * enc * 4 + 512
        ws = torch.empty(nbytes, dtype=torch.uint8, device=x.device)
        y = torch.empty(rows, desc.output_dim, dtype=torch.float32, device=x.device)
        prec = module._precision(ctx.needs_input_grad[0])
        N.check(lib.b200_mlp_forward(C.byref(desc), N.ptr(flat), N.ptr(x), N.ptr(y), rows, 1, prec, N.ptr(ws),
                                     ws.numel(), N.current_stream()), "b200_mlp_forward")
        ctx.save_for_backward(x, flat)
        ctx.ws, ctx.module, ctx.prec = ws, module, prec
        return y

    @staticmethod
    def backward(ctx, dy):
        x, flat = ctx.saved_tensors
        desc = ctx.module._desc
        lib = N.lib()
        dflat = torch.zeros_like(flat)
        dx = torch.empty_like(x) if ctx.needs_input_grad[0] else None
        N.check(lib.b200_mlp_backward(C.byref(desc), N.ptr(flat), N.ptr(x), N.ptr(dy.contiguous().float()),
                                      N.ptr(dflat), N.ptr(dx), x.shape[0], ctx.prec, N.ptr(ctx.ws),
                                      ctx.ws.numel(), N.current_stream()), "b200_mlp_backward")
        return dx, dflat, None


class IMLP(nn.Module):
    def __init__(self, input_dim, output_dim, hidden_dim=256, use_positional=True, positional_dim=10,
                 skip_layers=[4, 6], num_layers=8, verbose=True, use_tanh=True, apply_softmax=False):
        super().__init__()
        if apply_softmax:
            raise NotImplementedError("apply_softmax is unused by the stage-1 scripts and not provided")
        if use_positional and positional_dim < 1:
            # the reference builds a network on a 0-wide encoding (layer 0 sees no input); the library has no such
            # network and would otherwise build the one on the raw input instead
            raise N.B200Error(f"use_positional=True needs positional_dim >= 1 (got {positional_dim})")
        self.verbose, self.use_tanh = verbose, use_tanh
        self.skip_layers, self.num_layers = list(skip_layers), num_layers
        self.positional_dim, self.use_positional = positional_dim, use_positional
        self._desc = A.make_desc(input_dim, output_dim, hidden_dim, num_layers,
                                 positional_dim if use_positional else 0, self.skip_layers, use_tanh)
        self._w_off, self._b_off, self._total = A.mlp_layout(self._desc)
        # architectures of the stage-1 scripts with wgmma kernels (the library decides): 1 = mapping-shaped
        # (3 -> 256 x {2,4} -> 2, no encoding), 2 = atlas (2 -> PE 10 -> 256 x 6 -> 3, skips 4 and 7), 3 = alpha
        # (3 -> PE 5 -> 256 x 6 -> 1), 4 = position-encoded mapping (3 -> PE 1..10 -> 256 x {2,4} -> 2), 0 = fp32
        # kernels only
        self._tc_arch = max(0, int(N.lib().b200_mlp_tc_architecture(C.byref(self._desc))))
        # one flat fp32 buffer in the library's layout; the per-layer tensors are views of it
        self.flat = nn.Parameter(torch.zeros(self._total))
        for i, (k, n) in enumerate(A.layer_dims(self._desc)):
            bound = 1.0 / math.sqrt(k)
            with torch.no_grad():      # nn.Linear.reset_parameters: weight then bias, U(-1/sqrt(k), 1/sqrt(k))
                self.flat[self._w_off[i]:self._w_off[i] + k * n] = torch.empty(n, k).uniform_(-bound, bound).flatten()
                self.flat[self._b_off[i]:self._b_off[i] + n] = torch.empty(n).uniform_(-bound, bound)
        if self.verbose:
            print(f'Model has {sum(k * n + n for k, n in A.layer_dims(self._desc))} params')

    # ---- reference-compatible state dict: hidden.{i}.weight / hidden.{i}.bias
    def _views(self, flat):
        out = {}
        for i, (k, n) in enumerate(A.layer_dims(self._desc)):
            out[f"hidden.{i}.weight"] = flat[self._w_off[i]:self._w_off[i] + k * n].view(n, k)
            out[f"hidden.{i}.bias"] = flat[self._b_off[i]:self._b_off[i] + n]
        return out

    def state_dict(self, *args, **kwargs):
        return {k: v.detach().clone() for k, v in self._views(self.flat).items()}

    def load_state_dict(self, sd, strict=True):
        with torch.no_grad():
            for k, v in self._views(self.flat).items():
                if k in sd:
                    v.copy_(sd[k])
                elif strict:
                    raise KeyError(k)

    def _precision(self, input_needs_grad: bool) -> int:
        """Tensor cores (B200_PREC_TC: 2-term fp16 operands, fp32 accumulation — DESIGN.md §3) whenever the
        architecture has the fused kernels and the device is sm_90; `B200_IMLP_PRECISION=fp32|tc` overrides.  The
        mapping (codes 1, 4) / alpha kernels produce no input gradient (their inputs are pixel coordinates)."""
        import os
        want = os.environ.get("B200_IMLP_PRECISION", "auto")
        ok = self._tc_arch != 0 and bool(N.lib().b200_device_supports_tc()) and not (self._tc_arch != 2 and input_needs_grad)
        if want == "tc" and not ok:
            raise N.B200Error("B200_IMLP_PRECISION=tc: this IMLP has no tensor-core kernels on this device / call")
        return N.PREC_TC if (ok and want != "fp32") else N.PREC_FP32

    def forward(self, x):
        return _ImlpFunction.apply(x, self.flat, self)
