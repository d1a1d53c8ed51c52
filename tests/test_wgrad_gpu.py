"""The weight-gradient kernel (tc_wgrad_kernel: clusters of two CTAs, the N-side operand multicast to both) against
FLOAT64 autograd, with the tolerances of tests/test_tc_gpu.py.

* Stand-alone `IMLP` backward for every network, so every operand shape of the work list runs: 256x256 (hidden
  layers), 256x64 (positional-encoding chunk of atlas layer 0 and skip layer 4, PE mapping layer 0), 64x256 (output
  layers, computed transposed) and 64x64 (the atlas output layer's skip part, row steps split over the pair).  Row
  counts cover clusters with no row steps (1, 127, 129 rows: one or two tiles for dozens of clusters), partial shares,
  and just below / above one tile per cluster.  ||err||_F <= 3e-3 ||g||_F per weight, 1.5e-2 for the atlas.
* The fused step at the benchmarked configuration in both regimes (throughput set, random-init networks), every weight
  against float64 with the bounds of tests/test_tc_fullsize_gpu.py for that input: ||err||_F <= 8e-2 ||g||_F and
  max|err| <= 0.12 max|g|.  The random-init mapping makes its gradients ill-conditioned: there the tensor-core path
  sits 0.4 % (with the global rigidity term) to 2.5 % (without) from float64, one fp32 accumulator per unit of rows.
"""
import os

import numpy as np
import pytest
import torch

from b200 import _native as N
from b200 import atlas as A
from b200 import synth
from oracle import atlas_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _need_tc():
    if not N.lib().b200_device_supports_tc():
        pytest.skip("no sm_90 device")


def _cluster_rows():
    """Rows of one 128-row tile per cluster of two SMs, less and more one tile."""
    if not torch.cuda.is_available():
        return [8320, 8576]
    tiles = torch.cuda.get_device_properties(0).multi_processor_count // 2
    return [128 * (tiles - 1) - 5, 128 * (tiles + 1) + 3]


NETS = {  # name: (IMLP kwargs, oracle spec, input scale, tolerance)
    "mapping": (dict(input_dim=3, output_dim=2, use_positional=False, positional_dim=4, num_layers=6, skip_layers=[]),
                O.MlpSpec(3, 2, 256, False, 4, (), 6), 2.0, 3e-3),
    "mapping4": (dict(input_dim=3, output_dim=2, use_positional=False, positional_dim=2, num_layers=4, skip_layers=[]),
                 O.MlpSpec(3, 2, 256, False, 2, (), 4), 2.0, 3e-3),
    "atlas": (dict(input_dim=2, output_dim=3, use_positional=True, positional_dim=10, num_layers=8, skip_layers=[4, 7]),
              O.ATLAS_SPEC, 1.0, 1.5e-2),
    "alpha": (dict(input_dim=3, output_dim=1, use_positional=True, positional_dim=5, num_layers=8, skip_layers=[]),
              O.MlpSpec(3, 1, 256, True, 5, (), 8), 2.0, 3e-3),
    "pe_mapping": (dict(input_dim=3, output_dim=2, use_positional=True, positional_dim=4, num_layers=6, skip_layers=[]),
                   O.MlpSpec(3, 2, 256, True, 4, (), 6), 2.0, 3e-3),
}


@pytest.mark.parametrize("rows", [1, 127, 129] + _cluster_rows())
@pytest.mark.parametrize("which", list(NETS))
def test_imlp_weight_gradients(which, rows, monkeypatch):
    _need_tc()
    monkeypatch.setenv("B200_IMLP_PRECISION", "tc")
    from src.models.stage_1.implicit_neural_networks import IMLP
    kw, spec, scale, tol = NETS[which]
    net = IMLP(hidden_dim=256, verbose=False, **kw)
    assert net._tc_arch != 0
    torch.manual_seed(list(NETS).index(which) * 1000 + rows)
    params = O.init_mlp(spec)
    net.load_state_dict(O.state_dict_of(params))
    net = net.to(DEV)
    g = torch.Generator().manual_seed(rows)
    x = torch.rand(rows, spec.input_dim, generator=g) * scale - (scale - 1.0)
    w = torch.randn(rows, spec.output_dim, generator=g)
    (net(x.to(DEV)) * w.to(DEV)).sum().backward()
    p64 = [p.double().requires_grad_(True) for p in params]
    (O.mlp_forward(spec, p64, x.double()) * w.double()).sum().backward()
    views = net._views(net.flat.grad)
    errs = {}
    for i in range(len(params) // 2):
        t = p64[2 * i].grad
        errs[i] = float((views[f"hidden.{i}.weight"].cpu().double() - t).norm() / t.norm())
    assert max(errs.values()) <= tol, (which, rows, errs)


@pytest.mark.parametrize("with_global,it", [(True, 0), (False, 6000)])
def test_fused_step_weight_gradients_at_benchmark_shape(golden_dir, with_global, it):
    _need_tc()
    torch.set_num_threads(min(32, os.cpu_count() or 1))
    H, W, T, B = 432, 768, 80, 10000
    data = synth.throughput_set(H, W, T, seed=0)
    z = np.load(os.path.join(golden_dir, "params_seed1234.npz"))
    mp = [torch.from_numpy(z[f"map{i}"]) for i in range(12)]
    ap = [torch.from_numpy(z[f"atl{i}"]) for i in range(16)]
    inds = torch.randint(H * W * T, (B, 1), generator=torch.Generator().manual_seed(1))
    vid = A.DeviceVideo.from_reference_layout(data, DEV)
    tr = A.AtlasTrainer(vid, {"samples_batch": B}, precision=N.PREC_TC, device=DEV)
    tr.load_state(O.state_dict_of(mp), O.state_dict_of(ap))
    tr.indices.copy_(inds.reshape(-1))
    tr.loss_grad(with_global)
    torch.cuda.synchronize()
    got = [g.cpu().double() for w in ("mapping", "atlas") for g in tr.grad_views(w).values()]
    video64 = O.Video(**{k: v.double() if v.dtype == torch.float32 else v for k, v in data.items()})
    m64 = [p.double().requires_grad_(True) for p in mp]
    a64 = [p.double().requires_grad_(True) for p in ap]
    O.iteration_losses(video64, m64, a64, inds, it)["total"].backward()
    errs = {}
    for i, (g, p) in enumerate(zip(got, m64 + a64)):
        if p.dim() == 2:
            e = (g - p.grad).abs()
            errs[i] = (float(e.norm() / p.grad.norm()), float(e.max() / p.grad.abs().max()))
    bad = {i: e for i, e in errs.items() if e[0] > 8e-2 or e[1] > 0.12}
    assert not bad, (bad, errs)
