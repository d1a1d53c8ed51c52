"""`RAFT` (basic variant, the only one the reference's wrapper builds: raft_wrapper.py:17-20) with the
reference's module tree / state_dict keys and forward signature (src/models/stage_1/core/raft.py:28-148).
Inference only (the reference never trains it).  `args.mixed_precision` keeps the reference's meaning
(core/raft.py:99,110,131: encoders and update block under fp16 autocast, correlation in fp32): the
convolutions of those three sub-networks then run on the wgmma path (fp16 operands, fp32 accumulation,
fp32 tensors between layers); without it every convolution is the fp32 CUDA-core kernel."""
import contextlib

import torch
import torch.nn as nn

from b200 import _native as N
from b200 import nn as K
from src.models.stage_1.core.corr import AlternateCorrBlock, CorrBlock
from src.models.stage_1.core.extractor import BasicEncoder
from src.models.stage_1.core.update import BasicUpdateBlock
from src.models.stage_1.core.utils.utils import coords_grid


def corr_block_class(args, H8, W8, device_bytes):
    """The correlation block RAFT uses for feature maps of H8 x W8: `AlternateCorrBlock` when `args.alternate_corr` is
    set (the reference's switch) or when the all-pairs pyramid would take more than half of the device's memory
    (`device_bytes`; 4K frames need 89 GB), `CorrBlock` otherwise.  `device_bytes=None`: memory not known."""
    if getattr(args, "alternate_corr", False):
        return AlternateCorrBlock
    if device_bytes is not None and int(N.lib().b200_corr_pyramid_floats(H8, W8)) * 4 > device_bytes // 2:
        return AlternateCorrBlock
    return CorrBlock


class RAFT(nn.Module):
    def __init__(self, args):
        super().__init__()
        self.args = args
        if getattr(args, "small", False):
            raise NotImplementedError("RAFT-small is unreachable with the reference's arguments")
        self.hidden_dim = hdim = 128
        self.context_dim = cdim = 128
        args.corr_levels, args.corr_radius = 4, 4
        if not hasattr(args, "dropout"):
            args.dropout = 0
        if not hasattr(args, "alternate_corr"):
            args.alternate_corr = False
        self.fnet = BasicEncoder(output_dim=256, norm_fn='instance', dropout=args.dropout)
        self.cnet = BasicEncoder(output_dim=hdim + cdim, norm_fn='batch', dropout=args.dropout)
        self.update_block = BasicUpdateBlock(self.args, hidden_dim=hdim)
        self._graph_state = {}          # (fmap shape, iters, device, block) -> captured refinement loop + its buffers

    @contextlib.contextmanager
    def _autocast(self):
        if not getattr(self.args, "mixed_precision", False) or K.conv_precision() != "fp32":
            yield                      # an explicit global choice (b200.nn.set_conv_precision) wins
            return
        prev = K.set_conv_precision("tc")
        try:
            yield
        finally:
            K.set_conv_precision(prev)

    @torch.no_grad()
    def forward(self, image1, image2, iters=12, flow_init=None, upsample=True, test_mode=False):
        """core/raft.py:93-148 for a batch of B frame pairs (B, 3, H, W); every sample's flow has the bits of the
        same pair run alone."""
        image1 = (2 * (image1 / 255.0) - 1.0).contiguous()
        image2 = (2 * (image2 / 255.0) - 1.0).contiguous()
        with self._autocast():
            fmap1, fmap2 = self.fnet([image1, image2])
            cnet = self.cnet(image1)
        return self._refine(fmap1, fmap2, cnet, iters, flow_init, test_mode)

    @torch.no_grad()
    def forward_both(self, image1, image2, iters=12):
        """Flow 1->2 and 2->1 of one frame pair: forward_sequence on the two frames."""
        return self.forward_sequence(torch.cat([image1, image2]), iters)

    @torch.no_grad()
    def forward_sequence(self, images, iters=12, pad_to=None):
        """K + 1 consecutive frames (K + 1, 3, H, W) -> ((flow_low, flow_up) of the K forward flows k -> k + 1,
        (flow_low, flow_up) of the K backward flows k + 1 -> k), each (K, 2, ...).  fnet and cnet run once per frame
        (the reference's pre-pass, preprocess_optical_flow.py:29-30, encodes each interior frame four times), and the 2K
        refinements run as one batch in the captured graph.  Each flow is `forward(a, b, iters, test_mode=True)` bit
        for bit.  `pad_to`: refine a batch of 2 * pad_to flows (>= K; the extra ones repeat the last flow and are
        dropped), so that a shorter window reuses the graph, and its correlation buffer, of the full-length one."""
        k = images.shape[0] - 1
        if k < 1:
            raise ValueError("forward_sequence needs at least two frames")
        kp = k if pad_to is None else pad_to
        if kp < k:
            raise ValueError(f"pad_to={pad_to} is smaller than the {k} pairs given")
        x = (2 * (images / 255.0) - 1.0).contiguous()
        with self._autocast():
            fmaps = self.fnet(x)
            ctx = self.cnet(x)
        fmap1 = torch.cat([fmaps[:-1], fmaps[1:]])
        fmap2 = torch.cat([fmaps[1:], fmaps[:-1]])
        cnet = torch.cat([ctx[:-1], ctx[1:]])
        del fmaps, ctx                             # the refinement's peak memory holds only the batched copies
        if kp > k:
            fmap1, fmap2, cnet = (torch.cat([t, t[-1:].expand(2 * (kp - k), *t.shape[1:])]) for t in (fmap1, fmap2, cnet))
        lo, up = self._refine(fmap1, fmap2, cnet, iters, None, True)
        return (lo[:k], up[:k]), (lo[k:2 * k], up[k:2 * k])

    def _refine(self, fmap1, fmap2, cnet, iters, flow_init, test_mode):
        """core/raft.py:109-148 from the feature maps and the context encoder's output.  In test mode the `iters`
        refinement iterations (lookup -> update block -> coordinate update, ~100 launches each plus tensor glue) are
        captured once per geometry (batch included) in ONE CUDA graph and replayed: the correlation block's state
        (pyramids or feature-map levels), hidden state, context and coordinates live in buffers owned by this module."""
        use_graph = test_mode and getattr(self.args, "cuda_graph", True) and fmap1.is_cuda
        n, _, h8, w8 = fmap1.shape
        block = corr_block_class(self.args, h8, w8,
                                 torch.cuda.get_device_properties(fmap1.device).total_memory if fmap1.is_cuda else None)
        key = (tuple(fmap1.shape), int(iters), fmap1.device, block)
        st = self._graph_state.get(key) if use_graph else None
        corr_fn = block(fmap1.float(), fmap2.float(), radius=self.args.corr_radius,
                        out=st["corr"] if st is not None else None)
        net, inp = torch.split(cnet, [self.hidden_dim, self.context_dim], dim=1)
        net, inp = torch.tanh(net).contiguous(), torch.relu(inp).contiguous()
        coords0 = coords_grid(n, h8, w8).to(fmap1.device)
        coords1 = coords0.clone()
        if flow_init is not None:
            coords1 = coords1 + flow_init
        if use_graph:
            if st is None:
                # first call for this geometry: adopt the buffers, run the loop once eagerly (fills the weight-image
                # caches, so nothing is packed or allocated outside the graph pool during capture), then capture
                st = dict(corr=corr_fn.state if block is AlternateCorrBlock else corr_fn.pyramid, net=net.clone(),
                          inp=inp.clone(), c0=coords0.clone(), c1=coords1.clone())
                self._loop(corr_fn, st["net"].clone(), st["inp"], st["c0"], st["c1"].clone(), iters, True)
                torch.cuda.synchronize()
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    st["out"] = self._loop(corr_fn, st["net"], st["inp"], st["c0"], st["c1"], iters, True)
                st["graph"] = g
                self._graph_state[key] = st
            st["net"].copy_(net); st["inp"].copy_(inp); st["c0"].copy_(coords0); st["c1"].copy_(coords1)
            st["graph"].replay()
            flow_lo, flow_up = st["out"]
            return flow_lo.clone(), flow_up.clone()
        return self._loop(corr_fn, net, inp, coords0, coords1, iters, test_mode)

    def _loop(self, corr_fn, net, inp, coords0, coords1, iters, test_mode):
        flow_up, preds = None, []
        for it in range(iters):
            corr = corr_fn(coords1)
            flow = (coords1 - coords0).contiguous()
            with self._autocast():
                net, up_mask, delta_flow = self.update_block(net, inp, corr, flow)
            coords1 = coords1 + delta_flow
            if not test_mode or it == iters - 1:          # test mode returns only the last upsampled flow
                flow_up = K.convex_upsample((coords1 - coords0).contiguous(), up_mask)
                preds.append(flow_up)
        if test_mode:
            return coords1 - coords0, flow_up
        return preds
