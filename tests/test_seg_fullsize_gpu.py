"""Segmentation variant at the benchmarked geometry (80 x 432 x 768, 10 000 samples per trip, the configuration
`bench.py --workload seg` times) on the tensor-core path against oracle/seg_oracle.py: one trip on the same index batch
and parameters.  The two mapping networks are first pre-trained for one sweep on the GPU (as the script does for 100),
so that the rigidity Jacobians are the well-conditioned ones of a real run.

Bounds (measured values are printed; fp32 oracle = the reference's arithmetic):
  every loss term   rtol 1e-4 (measured <= 2e-6)          flow-row counts exact
  gradients         per network ||err||_F <= 5e-3 ||g||_F (tensor-core networks; measured 7.1e-4, 4.5e-4, 3.1e-4),
                    1e-4 (alpha network, fp32 kernels; measured 2.9e-6)
"""
import numpy as np
import pytest
import torch

from b200 import _native as N
from b200 import atlas as A
from b200 import seg as SG
from b200 import synth
from oracle import atlas_oracle as O
from oracle import seg_oracle as S

pytestmark = pytest.mark.gpu
DEV = "cuda"


def test_seg_trip_at_benchmark_size_matches_oracle():
    if not N.lib().b200_device_supports_tc():
        pytest.skip("needs sm_90")
    T, H, W, B = 80, 432, 768, 10000
    data = synth.throughput_set(H, W, T, seed=0)
    masks = (torch.rand(H, W, T, generator=torch.Generator().manual_seed(2)) < 0.4).float()
    vid = A.DeviceVideo.from_reference_layout(data, DEV)
    tr = SG.SegTrainer(vid, SG.pack_mask_frames(masks, DEV), None, precision=N.PREC_TC, device=DEV)
    torch.manual_seed(11)
    tr.init_like_reference()
    for which in ("mapping1", "mapping2"):
        tr.pretrain(which, T, H, W, 1)
    inds = torch.randint(H * W * T, (B, 1), generator=torch.Generator().manual_seed(3))
    tr.indices.copy_(inds.reshape(-1))
    tr.loss_grad(0)
    torch.cuda.synchronize()
    got = tr.loss_dict()
    nets = {k: [v.detach().cpu().clone().requires_grad_(True) for v in tr.param_views(k).values()] for k in SG.NETS}
    torch.set_num_threads(min(32, torch.get_num_threads()))
    terms = S.seg_iteration_losses(O.Video(**data), masks, nets, inds, 0)
    terms["total"].backward()
    rel = {k: abs(got[k] - float(v.detach())) / abs(float(v.detach())) for k, v in terms.items()}
    print("seg full-size loss errors:", {k: f"{e:.1e}" for k, e in rel.items()})
    assert max(rel.values()) <= 1e-4, rel
    jif = O.pixel_table(T, H, W)[:, inds]
    n_f = int(data["mask_fwd"][jif[1].squeeze(), jif[0].squeeze(), jif[2].squeeze(), 0].sum())
    n_b = int(data["mask_bwd"][jif[1].squeeze(), jif[0].squeeze(), jif[2].squeeze(), 0].sum())
    assert (got["n_fwd"], got["n_bwd"]) == (n_f, n_b)
    worst = {}
    for k in SG.NETS:
        num = sum(float((g.cpu().double() - p.grad.double()).pow(2).sum()) for g, p in zip(tr.grad_views(k).values(), nets[k]))
        den = sum(float(p.grad.double().pow(2).sum()) for p in nets[k])
        worst[k] = (num / den) ** 0.5
    print("seg full-size gradient errors (Frobenius, per network):", {k: f"{e:.1e}" for k, e in worst.items()})
    assert worst["alpha"] <= 1e-4 and max(worst[k] for k in ("mapping1", "mapping2", "atlas")) <= 5e-3, worst
