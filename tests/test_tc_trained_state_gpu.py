"""The fused tensor-core IMLP kernels of csrc/mlp_tc.cu on trained weights and at the edges of their gradient scale,
layer by layer against float64 with the checks and the bound of test_tc_layers_gpu.py (its docstring states them).

The backward stores every dZ as a 2-term fp16 split of s_g dZ, one power of two per network: s_g = 2^(13 - e) with
max |dy| < 2^e, e clamped to [-60, 60] (`grad_scales`).  So max |dy| s_g < 2^13 and an inner dZ keeps its 22-bit
split while it stays below 8 max |dy| (hi saturates at 65504 = 2^16 - 32).  Initial weights sit far inside that
(inner dZ at most 0.07 max |dy|); trained weights come closer, and the cases here measure how close:

  trained trip      the parameters of the 10 001-iteration oracle run (tests/golden/quality_oracle.npz) on the video
                    they were trained on (synth.quality_set(432, 768, 80, seed=0)), B = 10 000: the fused stage-1 trip
                    with the global term (it = 0) and without it (it = 6000), and rank 0 / rank 1 of a 2-way frame
                    shard, on a 0xFF workspace (check_atlas_trip: images, dead tiles, dW, d_uv)
  trained pretrain  the pre-training trip on the trained mapping, B = 129 and 10 000
  grown weights     the stand-alone IMLP call of the six tensor-core networks, 129 and 3 * 132 * 128 - 50 rows, on
                    initial weights rescaled so that the float64 dZ of layer 0 reaches 1, 3 and 6 max |dy| (asserted on
                    the host) while the forward output stays what it was: the 256 hidden columns of every layer past
                    the first times alpha, layer 0, every bias and every encoding column times alpha^(l - L + 1) (ReLU
                    is positively homogeneous, so every mask and y is unchanged and dZ_l grows by alpha^(L - 1 - l))
  scale edges       the stand-alone backward of the trained mapping and atlas on a chosen dy: all zero (e = 0, zero
                    gradients and images), max |dy| = 2^-3 exactly and the float below it, one row 2^20 and 2^40 times
                    the others (the other rows' dZ fall into fp16 subnormals and must meet the bound with its 2^-24
                    floor), max |dy| = 2^59 and 2^-59 (just inside the clamp) and 2^-64 (below it: s_g stops at 2^73)

Every case checks that no hi term of any image is +-65504, prints max |hi + lo| / 65504 of each activation, encoding
and dZ image and the largest inner dZ over max |dy| s_g (`pytest -s`), and asserts that ratio is at most 8.  The
gradient scale is recomputed on the host from the gmax word the call used; the edge cases also state the e they
expect.  The module's peak device memory is printed at its end: 6.3 GiB allocated; its 58 cases take about 33 s,
15 s of which build the video on the CPU (H100 80GB HBM3, 700 W power limit).
"""
import math
import os

import numpy as np
import pytest
import torch

from b200 import _native as N
from b200 import atlas as A
from b200 import synth
from oracle import atlas_oracle as O
from tc_images_common import (DEV, HID, S_ACT, Net, _need_tc, desc_dims, encoding_ref, f64, host_counts, run_trip,
                              small_data, wg_units)  # noqa: F401  (wg_units: a fixture)
from test_atlas_eval_gpu import _unflat
from test_tc_layers_gpu import (B_SMALL, FULL, NETS, _init_flat, _seed, _trainer, check_atlas_trip, check_imlp,
                                check_pretrain_trip)

pytestmark = pytest.mark.gpu

F16_MAX = 65504.0
ENVELOPE = 8.0                   # inner dZ / (max |dy| s_g) the design keeps below the fp16 range
FIXTURE = "quality_oracle.npz"


def _f32(word):
    return float(np.int32(word).view(np.float32))


def headroom(label, im, net, s_g, word):
    """Prints max |hi + lo| / 65504 of every image of `im` and the inner dZ over max |dy| s_g per layer; asserts the
    largest of those ratios is within ENVELOPE and returns it."""
    def top(img):
        return float((f64(img[0]) + f64(img[1])).abs().max()) if img[0].numel() else 0.0

    L = net.L
    acts = [top(im.act(l)) / F16_MAX for l in range(L - 1)]
    slots = range(0 if net.pe else 1, L - 1)          # the plain mapping keeps dZ_0 on chip
    dz = {l: top(im.dz(l)) for l in slots}
    scale = _f32(word) * s_g
    inner = {l: v / scale if scale else 0.0 for l, v in dz.items()}
    fmt = lambda v: " ".join(f"{x:.3g}" for x in v)
    enc = f", encoding {top(im.pe()) / F16_MAX:.3g}" if net.pe else ""
    print(f"{label}: max |hi + lo| / 65504 of h0..h{L - 2} {fmt(acts)}; of dZ{slots[0]}..dZ{L - 2} "
          f"{fmt(v / F16_MAX for v in dz.values())}; dZ output {top(im.dzl()) / F16_MAX:.3g}{enc}; "
          f"inner dZ / (max |dy| s_g) {fmt(inner.values())}")
    largest = max(inner.values())
    assert largest <= ENVELOPE, f"{label}: an inner dZ is {largest:.3g} max |dy| s_g, past the design's {ENVELOPE}"
    return largest


@pytest.fixture(scope="module", autouse=True)
def peak_memory():
    yield
    if torch.cuda.is_available():
        print(f"peak device memory of the module: {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")


# ---------------------------------------------------------------------------------------------------------------
# the trained state
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def trained_state(golden_dir):
    fx = np.load(os.path.join(golden_dir, FIXTURE))
    assert tuple(int(v) for v in fx["video"]) == (FULL["T"], FULL["H"], FULL["W"]) and int(fx["iters"]) > 10000
    return _unflat(O.MAPPING_SPEC, fx["mapping_params"]), _unflat(O.ATLAS_SPEC, fx["atlas_params"])


@pytest.fixture(scope="module")
def trained_video(trained_state):
    """The video the fixture's parameters were trained on, an index batch and a whole-video trainer."""
    _need_tc()
    T, H, W, B = FULL["T"], FULL["H"], FULL["W"], FULL["B"]
    torch.set_num_threads(min(32, os.cpu_count() or 1))
    data = synth.quality_set(H, W, T, seed=0)
    data.pop("clean")
    inds = torch.randint(H * W * T, (B,), generator=torch.Generator().manual_seed(7))
    return data, inds, _trainer(data, B, state=trained_state)


@pytest.mark.parametrize("it", [0, 6000])
def test_trained_fused_trip(trained_video, it, wg_units):
    """The whole video: with the global rigidity term at it = 0, without it at it = 6000."""
    data, inds, tr = trained_video
    T, H, W = FULL["T"], FULL["H"], FULL["W"]
    wg = tr.uses_global(it)
    assert wg == (it == 0)
    tr.indices.copy_(inds)
    run_trip(tr, wg)
    label = f"trained fused trip, it {it}"
    keep = []
    check_atlas_trip(tr, wg, host_counts(inds, data, 0, T, H, W), wg_units, label, keep=keep)
    for which, im, s_g, word in keep:
        headroom(f"{label}, {which}", im, im.net, s_g, word)


@pytest.mark.parametrize("rank", [0, 1])
def test_trained_shard_trip(trained_video, trained_state, rank, wg_units):
    """Rank 0 and the last rank of a 2-way frame shard, with the global term."""
    data, inds, _ = trained_video
    T, H, W, B = FULL["T"], FULL["H"], FULL["W"], FULL["B"]
    t0, t1 = A.frame_range(rank, 2, T)
    tr = _trainer(data, B, t0, t1, state=trained_state)
    tr.indices.copy_(inds)
    run_trip(tr, True)
    label = f"trained trip, 2-way shard, rank {rank}"
    keep = []
    check_atlas_trip(tr, True, host_counts(inds, data, t0, t1, H, W), wg_units, label, keep=keep)
    for which, im, s_g, word in keep:
        headroom(f"{label}, {which}", im, im.net, s_g, word)


@pytest.mark.parametrize("B", [129, 10000])
def test_trained_pretrain_trip(trained_state, B, wg_units):
    _need_tc()
    data, _ = small_data()
    tr = _trainer(data, B_SMALL, state=trained_state)
    label = f"trained pre-training trip, B {B}"
    im, s_g, word = check_pretrain_trip(tr, B, wg_units, label)
    headroom(label, im, im.net, s_g, word)


# ---------------------------------------------------------------------------------------------------------------
# stand-alone calls on grown weights
# ---------------------------------------------------------------------------------------------------------------
GROWTH = [1.0, 3.0, 6.0]
GROWN_ROWS = [129, 3 * 132 * 128 - 50]


def _bias(net, l, flat):
    return flat[net.b_off[l]:net.b_off[l] + net.dims[l][1]]


def dz_chain(net, flat, x, dy):
    """float64 forward and backward of `net` with parameters `flat`: the dZ of layers 0 .. L-2 (host masks)."""
    L = net.L
    W = [net.weight(l, flat).double() for l in range(L)]
    b = [_bias(net, l, flat).double() for l in range(L)]
    enc = encoding_ref(net, x)[:, :net.enc] / S_ACT if net.pe else x.double()
    masks, h = [], None
    for l in range(L):
        inp = enc if l == 0 else (torch.cat((h, enc), 1) if net.skip[l] else h)
        z = inp @ W[l].T + b[l]
        if l < L - 1:
            masks.append(z > 0)
            h = torch.relu(z)
    dz = dy.double() * (1 - torch.tanh(z) ** 2)
    out = [None] * (L - 1)
    for l in range(L - 1, 0, -1):
        dz = (dz @ W[l][:, :HID]) * masks[l - 1]
        out[l - 1] = dz
    return out


def grown(net, flat, alpha):
    """`flat` with the dZ of layer l grown by alpha^(L - 1 - l) and the forward output unchanged: layer l's output
    scaled by s_l = alpha^(l - L + 1), so its hidden inputs by alpha and its bias and encoding inputs by s_l."""
    f = flat.clone()
    L = net.L
    for l in range(L):
        s = alpha ** (l - (L - 1))
        w = net.weight(l, f)
        if l == 0:
            w.mul_(s)
        else:
            w[:, :HID].mul_(alpha)
            w[:, HID:].mul_(s)
        _bias(net, l, f).mul_(s)
    return f


@pytest.mark.parametrize("rows", GROWN_ROWS)
@pytest.mark.parametrize("growth", GROWTH)
@pytest.mark.parametrize("which", list(NETS))
def test_grown_weights(which, growth, rows, wg_units):
    """The stand-alone IMLP call where the float64 dZ of layer 0 is `growth` times max |dy|."""
    _need_tc()
    dims, xs, xo = NETS[which]
    g = torch.Generator().manual_seed(_seed(f"grown {which}/{rows}"))
    net = Net(dims, None)
    init = _init_flat(net, g)
    x = (torch.rand(rows, net.in_dim, generator=g) * xs + xo).to(DEV)
    dy = torch.randn(rows, net.out, generator=g).to(DEV)
    gmax = float(dy.abs().max())
    g0 = float(dz_chain(net, init, x, dy)[0].abs().max()) / gmax
    alpha = (growth / g0) ** (1.0 / (net.L - 1))
    net.flat = grown(net, init, alpha)
    chain = [float(d.abs().max()) / gmax for d in dz_chain(net, net.flat, x, dy)]
    assert abs(chain[0] / growth - 1) < 0.02, (which, growth, chain)
    assert max(chain) <= ENVELOPE, (which, growth, chain)
    label = f"{which} grown to {growth} (alpha {alpha:.3g}; float64 dZ0..dZ{net.L - 2} / max |dy| " \
            f"{' '.join(f'{c:.3g}' for c in chain)}), rows {rows}"
    res = check_imlp(net, x, dy, wg_units, label)
    headroom(label, res["im"], net, res["s_g"], res["word"])


# ---------------------------------------------------------------------------------------------------------------
# gradient-scale edges
# ---------------------------------------------------------------------------------------------------------------
EDGE_ROWS = 3 * 132 * 128 - 50
K_POW2 = -3


def _below(v):
    return float(np.nextafter(np.float32(v), np.float32(0)))


def edge_dy(case, rows, out, g):
    """dy of one edge case and the e of `grad_scales` it must give (clamped)."""
    dy = torch.randn(rows, out, generator=g)
    unit = dy / dy.abs().max()                         # max |unit| = 1 exactly
    if case == "zero":
        return torch.zeros(rows, out), 0
    if case == "pow2":
        return unit * 2.0 ** K_POW2, K_POW2 + 1
    if case == "below_pow2":
        m = _below(2.0 ** K_POW2)
        return (unit * 2.0 ** K_POW2).clamp(-m, m), K_POW2
    if case.startswith("outlier"):
        dy[rows // 2] *= 2.0 ** int(case[7:])
        return dy, math.frexp(float(dy.abs().max()))[1]
    k = {"max_2^59": 59, "max_2^-59": -59, "below_clamp": -64}[case]
    return unit * 2.0 ** k, max(-60, min(60, k + 1))


@pytest.fixture(scope="module")
def trained_nets(trained_state):
    """The trained mapping and atlas as Nets (flat parameters on the device)."""
    _need_tc()
    tr = A.AtlasTrainer(None, precision=N.PREC_TC, device=DEV)
    tr.load_state(*trained_state)
    return {w: Net(desc_dims(tr.descs[w]), tr.params[tr.net_slice(w)].clone()) for w in ("mapping", "atlas")}


@pytest.mark.parametrize("case", ["zero", "pow2", "below_pow2", "outlier20", "outlier40", "max_2^59", "max_2^-59",
                                  "below_clamp"])
@pytest.mark.parametrize("which", ["mapping", "atlas"])
def test_grad_scale_edges(trained_nets, which, case, wg_units):
    """The stand-alone IMLP call of a trained network on a chosen dy: checks (a) to (d), s_g from the expected e."""
    net = trained_nets[which]
    _, xs, xo = NETS[which]
    g = torch.Generator().manual_seed(_seed(f"edge {which}/{case}"))
    x = (torch.rand(EDGE_ROWS, net.in_dim, generator=g) * xs + xo).to(DEV)
    dy, e = edge_dy(case, EDGE_ROWS, net.out, g)
    dy = dy.to(DEV)
    label = f"trained {which}, dy {case}"
    res = check_imlp(net, x, dy, wg_units, label)
    assert res["s_g"] == 2.0 ** (13 - e), (label, res["s_g"], e)
    im = res["im"]
    if case == "zero":
        assert res["word"] == 0
        assert torch.count_nonzero(_gradients(net, res["grads"])) == 0, f"{label}: a gradient is not zero"
        imgs = [im.dzl()] + [im.dz(l) for l in range(0 if net.pe else 1, net.L - 1)]
        assert all(torch.count_nonzero(t) == 0 for img in imgs for t in img), f"{label}: a dZ image is not zero"
        if net.atlas:
            assert torch.count_nonzero(res["d_in"]) == 0, f"{label}: d_in is not zero"
        return
    headroom(label, im, net, res["s_g"], res["word"])


def _gradients(net, grads):
    """Every weight and bias gradient of `net` in the flat block `grads`."""
    return torch.cat([net.weight(l, grads).flatten() for l in range(net.L)] +
                     [grads[net.b_off[l]:net.b_off[l] + net.dims[l][1]] for l in range(net.L)])
